"""Multinomial sampling (sample_max = 0) on the device: the sampler kernel op by op (gvd_op_reduce_sample) against float64 and the
definition in sample_ref.py, its distribution, and the whole decode loop (gvd_decode_sample, the nn.Module surface) against the oracle with
the same counter-based noise.

The noise seeds of the model-level cases are chosen so that no oracle key has a near-tie (top-2 gap < 1e-3) at any step; the comparison
still stops at the first step that would have one."""
import math
import warnings

import numpy as np
import pytest
import torch
from scipy import stats

import sample_ref as SR
from cases import CASES, build_case
from gvd_b200 import capi
from test_gpu_decode_ops import E_, T_, _PickOut, _gen, _rup

pytestmark = pytest.mark.gpu

NAN = float("nan")
TOL = 1e-4


@pytest.fixture(autouse=True)
def _restore_backend():
    prev = capi.get_backend()
    yield
    capi.set_backend(prev)
    capi.profile_enable(False)


# ------------------------------------------------------------------------------------------------------------ a. the sampler kernel
def _launch(part, bias, V, tau, seed, step, embed=None, image=True):
    B = part.shape[1]
    o = _PickOut(B, image=image and embed is not None)
    kw = o.args(embed) if embed is not None else dict(seq=o.seq[:, T_], logp=o.logp[:, T_])
    capi.op_reduce_sample(part, bias, V, tau, seed, step, o.it, **kw)
    return o


def _reference(logits32, tau, seed, step, rows=None):
    """float64 keys, token and log-probability from the float32 logits the kernel forms (same summation order)."""
    l64 = logits32.double().numpy()
    B, V = l64.shape
    g = SR.gumbel_noise(seed, np.arange(B) if rows is None else rows, step, V)
    with np.errstate(invalid="ignore"):
        key = l64 / tau + g
        srt = np.sort(key, axis=1)
        gap = srt[:, -1] - srt[:, -2]
        tok = np.argmax(key, axis=1)
        m = l64.max(axis=1, keepdims=True)
        lse = m[:, 0] + np.log(np.exp(l64 - m).sum(axis=1))
    return tok, l64[np.arange(B), tok] - lse, gap


_VOCABS = [2, 7, 2048, 2049, 4905, 5120, 5121, 6144]          # 2048|2049 and 5120|5121: reduce_sample_kernel<2|5|6> boundaries


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("V", _VOCABS)
def test_sampler_matches_float64_definition(V, S, tau):
    """Token = argmax(l / tau + g) of the fp64 definition on every row whose fp64 top-2 key gap exceeds 1e-5 (at most 1 % excluded),
    log-probability (untempered) within 1e-5, xt = ReLU(embed[token]) bitwise and its fp16x3 image.  S = 1 without bias is the plain loop
    path (logits already hold the bias), S = 3 with bias the split-K path."""
    B, step, seed = 128, 3, 0x5EED0000 + V * 7 + S
    g = _gen(V * 10 + S)
    ldp = _rup(V, 4) + 4
    part = torch.randn(S, B, ldp, generator=g) / S ** 0.5
    bias = torch.randn(V, generator=g) if S > 1 else None
    logits = part[0, :, :V].clone()
    for s in range(1, S):                                  # the kernel's order: ascending s, then the bias
        logits += part[s, :, :V]
    if bias is not None:
        logits += bias
    embed = torch.randn(V, E_, generator=g).cuda()
    o = _launch(part.cuda(), bias.cuda() if bias is not None else None, V, tau, seed, step, embed)
    want_tok, want_lp, gap = _reference(logits, tau, seed, step)
    rows = np.nonzero(gap > 1e-5)[0]
    assert rows.size >= 0.99 * B, rows.size
    o.check("reduce_sample V=%d S=%d tau=%g" % (V, S, tau), want_tok, want_lp, embed, 1e-5, rows=rows)
    if V >= 2048:                                          # a draw, not the argmax of the logits
        assert (want_tok != logits.numpy().argmax(1)).mean() > 0.05


def test_sampler_edge_rows():
    """-inf words are never drawn (also when their key would win); a row of -inf or of NaN yields token 0; equal keys (two +inf logits,
    in the same thread, across warps and at the end of the row) go to the lower index; any word, UNK included, is drawable."""
    V, B = 6144, 24
    rs = np.random.RandomState(3)
    x = rs.standard_normal((B, V)).astype(np.float32)
    want = np.zeros(B, np.int64)
    x[0] = -np.inf
    x[1] = np.nan
    for r, (j, k) in enumerate([(7, 3000), (100, 100 + 1024), (6142, 6143), (0, 6143)]):
        x[2 + r, j] = x[2 + r, k] = np.inf
        want[2 + r] = min(j, k)
    dominant = [0, 1, 31, 32, 1023, 1024, 2047, 2048, 4904, 5119, 5120, 6143, 3333, 77]
    for r, w in enumerate(dominant):
        x[6 + r, w] = 40.0
        want[6 + r] = w
    x[20:, :] = rs.standard_normal((4, V)) * 0.1           # flat rows with masked words, one of which would otherwise dominate
    masked = rs.choice(V, 300, replace=False)
    x[20:, 17] = 60.0
    masked = np.union1d(masked, [0, 17, V - 1])
    x[20:, masked] = -np.inf
    embed = torch.randn(V, E_, generator=_gen(4)).cuda()
    part = torch.from_numpy(x).reshape(1, B, V).cuda()
    for step in range(4):
        o = _launch(part, None, V, 1.0, 99, step, embed)
        tok_ref, _, gap = _reference(torch.from_numpy(x[20:]), 1.0, 99, step, rows=np.arange(20, B))
        want[20:] = tok_ref
        assert (gap > 1e-5).all()
        o.check("edge rows, step %d" % step, want, None, embed, None)
        assert not np.isin(o.it.cpu().numpy()[20:], masked).any()


def test_sampler_rejects_bad_arguments():
    B = 4
    it = torch.full((B,), -1, dtype=torch.int64, device="cuda")
    for V in (1, 6145):
        with pytest.raises(capi.GvdError):
            capi.op_reduce_sample(torch.zeros(1, B, V + 3, device="cuda"), None, V, 1.0, 0, 0, it)
    for tau in (0.0, -1.0, NAN, float("inf")):
        with pytest.raises(capi.GvdError):
            capi.op_reduce_sample(torch.zeros(1, B, 304, device="cuda"), None, 301, tau, 0, 0, it)
    torch.cuda.synchronize()
    assert bool((it == -1).all())


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
def test_sampler_distribution(tau):
    """128 rows x 160 steps of one fixed 7-word row (one word masked): Pearson chi-square against softmax(l / tau) with p > 1e-6 (fixed
    seeds: deterministic), the masked word never drawn, and rows b, b + 1 of the same step agreeing as often as independent draws do
    (sum p^2, within 5 sigma) — the row index is part of the counter."""
    B, steps, V = 128, 160, 7
    lvec = np.array([1.0, 0.5, -np.inf, 2.0, 0.0, -1.0, 1.5], np.float32)
    part = torch.from_numpy(np.tile(lvec, (B, 1))).reshape(1, B, V)
    part = torch.cat((part, torch.zeros(1, B, 1)), dim=2).cuda()
    toks = []
    for t in range(steps):
        o = _launch(part, None, V, tau, 20260 + int(tau * 10), t)
        toks.append(o.it)
    tok = torch.stack(toks).cpu().numpy()                  # [steps, B]
    p = np.exp(lvec.astype(np.float64) / tau)
    p /= p.sum()
    counts = np.bincount(tok.ravel(), minlength=V)
    assert counts[2] == 0
    live = p > 0
    chi = stats.chisquare(counts[live], counts.sum() * p[live])
    print("tau=%g counts=%s expected=%s chi2 p=%.3g" % (tau, counts.tolist(), np.round(counts.sum() * p).tolist(), chi.pvalue))
    assert chi.pvalue > 1e-6
    q = float((p ** 2).sum())
    n = steps * (B - 1)
    agree = int((tok[:, :-1] == tok[:, 1:]).sum())
    assert abs(agree - n * q) <= 5 * math.sqrt(n * q * (1 - q)), (agree, n * q)


# ------------------------------------------------------------------------------------------------------------ b. the decode loop
# noise seed per (case, temperature): no near-tie of the oracle's keys at any step
_SEEDS = {("greedy_T10_B4", 0.7): 107, ("greedy_T10_B4", 1.0): 110, ("greedy_T10_B4", 1.5): 1115,
          ("greedy_small_B5", 0.7): 107, ("greedy_small_B5", 1.0): 110, ("greedy_small_B5", 1.5): 115,
          ("greedy_T480_B2", 0.7): 107, ("greedy_T480_B2", 1.0): 1110, ("greedy_T480_B2", 1.5): 115}
_B100 = dict(kind="greedy", B=100, opt=dict(t_attn_size=10), input_seed=4242)
_B100_ROWS = [0, 13, 27, 41, 55, 69, 83, 99]
_cache = {}


def _module(opt, sd):
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    m.load_state_dict(sd)
    return m.cuda().eval()


def _case(name, case=None, rows=None):
    """(opt, state_dict, inputs, module, oracle prologue features of `rows`), built once per case."""
    if name not in _cache:
        import gvd_oracle as O
        opt, sd, inp = build_case(case or CASES[name])
        sub = inp if rows is None else {k: v[rows] for k, v in inp.items()}
        feats = O.prologue(sd, opt, sub["segs_feat"], sub["ppls"], sub["num"], sub["ppls_feat"], sub["sample_idx"], sub["pnt_mask"])
        _cache[name] = (opt, sd, inp, _module(opt, sd), feats)
    return _cache[name]


_KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


def _native_sample(model, inp, seed, tau):
    nm = model._native_model()
    B, T = inp["segs_feat"].shape[:2]
    dev = {k: inp[k].cuda() for k in _KEYS}
    nm.prologue(*(dev[k] for k in _KEYS))
    out = nm.decode_sample(B, T, dev["pnt_mask"], seed, tau)
    torch.cuda.synchronize()
    return [o.cpu() for o in out]


def _compare_with_oracle(got, opt, sd, inp, feats, tau, seed, rows):
    seq, logp, att2 = got
    oseq, ologp, oatt2, _, gaps = SR.sample_multinomial(sd, opt, inp, tau, SR.noise_fn(seed, rows, opt.vocab_size), feats=feats)
    k = int(np.argmax(gaps < 1e-3)) if (gaps < 1e-3).any() else opt.seq_length
    assert k == opt.seq_length, "a near-tie of the oracle keys at step %d: choose another seed" % k
    assert torch.equal(seq[:, :k], oseq[:, :k]), (seq, oseq)
    assert float((logp[:, :k] - ologp[:, :k]).abs().max()) <= TOL
    assert float((att2[:, :k].double() - oatt2[:, :k].double()).abs().max()) <= TOL
    assert torch.equal(att2[:, :k] == -1e8, oatt2[:, :k] == -1e8)
    return oseq


@pytest.mark.parametrize("backend", [923, 3, 0])
@pytest.mark.parametrize("tau", [0.7, 1.0, 1.5])
@pytest.mark.parametrize("name", ["greedy_T10_B4", "greedy_small_B5", "greedy_T480_B2"])
def test_decode_sample_matches_oracle(name, tau, backend):
    """The three loop paths (923: split-K product + sampler on the partial planes; 3: tensor-core head + sampler writing xt; 0: CUDA-core
    head, the core step embeds the token) against sample_multinomial with the same noise: tokens equal, log-probabilities (untempered)
    and attention logits within 1e-4."""
    capi.set_backend(backend)
    opt, sd, inp, model, feats = _case(name)
    seed = _SEEDS[(name, tau)]
    got = _native_sample(model, inp, seed, tau)
    B = inp["ppls"].shape[0]
    oseq = _compare_with_oracle(got, opt, sd, inp, feats, tau, seed, np.arange(B))
    assert len(np.unique(oseq.numpy())) > opt.seq_length


def test_decode_sample_full_batch():
    """B = 100, T = 10 (the benchmark's batch): 8 clips spread over the batch against the oracle, each with the noise of its row in the
    full batch."""
    opt, sd, inp, model, feats = _case("B100", _B100, _B100_ROWS)
    got = _native_sample(model, inp, 110, 1.0)
    rows = np.array(_B100_ROWS)
    sub = {k: v[rows] for k, v in inp.items()}
    _compare_with_oracle([o[rows] for o in got], opt, sd, sub, feats, 1.0, 110, rows)
    assert int(got[0].min()) >= 0 and int(got[0].max()) < opt.vocab_size


def test_graph_replay_and_interleaving():
    """A replay of the captured loop equals the kernel-by-kernel enqueue (stage profiler on) bit for bit, for two seeds that give different
    tokens (a new seed replays the same graph: the parameter block is copied in first); greedy, sample, greedy leaves the greedy outputs
    bit-identical to the greedy run before."""
    opt, sd, inp, model, _ = _case("greedy_small_B5")
    nm = model._native_model()
    B, T = inp["segs_feat"].shape[:2]
    dev = {k: inp[k].cuda() for k in _KEYS}
    nm.prologue(*(dev[k] for k in _KEYS))
    greedy0 = [o.clone() for o in nm.decode_greedy(B, T, dev["pnt_mask"])]
    got = {}
    for seed in (11, 12):
        replay = [o.clone() for o in nm.decode_sample(B, T, dev["pnt_mask"], seed, 0.8)]
        torch.cuda.synchronize()
        capi.profile_enable(True)
        direct = nm.decode_sample(B, T, dev["pnt_mask"], seed, 0.8)
        torch.cuda.synchronize()
        capi.profile_enable(False)
        for a, b in zip(replay, direct):
            assert torch.equal(a, b), seed
        got[seed] = replay
    assert not torch.equal(got[11][0], got[12][0])
    again = nm.decode_sample(B, T, dev["pnt_mask"], 11, 0.8)
    greedy1 = nm.decode_greedy(B, T, dev["pnt_mask"])
    torch.cuda.synchronize()
    for a, b in zip(again, got[11]):
        assert torch.equal(a, b)
    for a, b in zip(greedy1, greedy0):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------ c. the module surface
def _forward(model, inp, eval_opt):
    dev = {k: v.cuda() for k, v in inp.items()}
    d = torch.zeros(inp["ppls"].shape[0], dtype=torch.uint8, device="cuda")
    with torch.no_grad():
        out = model(dev["segs_feat"], d, d, dev["num"], dev["ppls"], d, d, dev["ppls_feat"], d, dev["sample_idx"], dev["pnt_mask"], "sample",
                    eval_opt)
    torch.cuda.synchronize()
    return out


def test_module_seeding_and_errors():
    """forward(..., 'sample', {'sample_max': 0}): the per-call seed comes from torch's default generator, so torch.manual_seed reproduces a
    call and successive calls differ; the returned triple has the greedy shapes; a temperature that is not finite and > 0 raises ValueError;
    train mode raises GvdError."""
    opt, sd, inp, model, _ = _case("greedy_small_B5")
    eo = {"sample_max": 0, "beam_size": 1, "temperature": 1.2}
    torch.manual_seed(5)
    a = _forward(model, inp, eo)
    b = _forward(model, inp, eo)
    torch.manual_seed(5)
    c = _forward(model, inp, eo)
    assert len(a) == 3 and a[0].shape == (5, opt.seq_length) and a[0].dtype == torch.int64
    assert a[1].shape == (5, opt.seq_length, opt.num_sampled_frm * opt.num_prop_per_frm)
    for x, y in zip(a, c):
        assert torch.equal(x, y)
    assert not torch.equal(a[0], b[0])
    torch.manual_seed(5)
    seed = int(torch.randint(0, 2 ** 62, (1,)))                 # the draw _sample makes
    seq, logp, att2 = _native_sample(model, inp, seed, 1.2)
    assert torch.equal(seq, a[0].cpu()) and torch.equal(att2, a[1].cpu())
    for tau in (0.0, -1.0, NAN, float("inf")):
        with pytest.raises(ValueError):
            _forward(model, inp, {"sample_max": 0, "beam_size": 1, "temperature": tau})
    model.train()
    try:
        with pytest.raises(capi.GvdError):
            _forward(model, inp, eo)
    finally:
        model.eval()


def test_module_dispatch_order():
    """The reference's order (model.py:501, 570-578): beam_size > 1 is beam search whatever sample_max is; the transformer captioner decodes
    greedily whatever sample_max is."""
    opt, sd, inp, model, _ = _case("greedy_small_B5")
    beam0 = _forward(model, inp, {"sample_max": 0, "beam_size": 3})
    beam1 = _forward(model, inp, {"sample_max": 1, "beam_size": 3})
    for x, y in zip(beam0, beam1):
        assert torch.equal(x, y)
    opt, sd, inp = build_case(CASES["tfm_greedy_small_B5"])
    tfm = _module(opt, sd)
    s0 = _forward(tfm, inp, {"sample_max": 0, "beam_size": 1, "temperature": 0.5})
    s1 = _forward(tfm, inp, {"sample_max": 1, "beam_size": 1})
    for x, y in zip(s0, s1):
        assert torch.equal(x, y)
