"""Vocabularies above 6144 words on the device: the sliced vocabulary tail (gvd_op_reduce_pick_split) op by op against float64, the greedy
rule's special rows and the existing tails, and every decode entry point of the top-down and transformer captioners against the oracle and
the reference's fixtures (tests/golden/vocab_cases.py).  Bars as tests/test_gpu_parity.py: token ids bit-exact, log-probs / logits /
losses within 1e-4; op level: log-probs within 1e-5, xt and its fp16x3 image bitwise."""
import warnings

import numpy as np
import pytest
import torch

import gvd_oracle as O
import sample_ref as SR
from cases import build_case, load_fixture, subsample
from gvd_b200 import capi
from sampler_ref import pick_reference, special_rows
from test_gpu_decode_ops import E_, T_, _PickOut, _exact_operands, _gen, _rup
from vocab_cases import VOCAB_CASES as CASES

pytestmark = pytest.mark.gpu
TOL = 1e-4
KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


@pytest.fixture(autouse=True)
def _restore_backend():
    b = capi.get_backend()
    yield
    capi.set_backend(b)
    capi.profile_enable(False)


# ------------------------------------------------------------------------------------------------------------ the tail, op by op
def _planes(V, S, B, seed, with_bias=True, unk_boost=0.0):
    """Random planes [S, B, ldp] (NaN beyond V, as the products leave them) + bias (its last word raised by unk_boost), and the float32
    logits in the kernel's order."""
    g = _gen(seed)
    ldp = _rup(V, 4) + 4
    part = torch.randn(S, B, ldp, generator=g) / S ** 0.5
    part[:, :, V:] = float("nan")
    bias = torch.randn(V, generator=g) if with_bias else None
    if bias is not None:
        bias[V - 1] += unk_boost
    logits = part[0, :, :V].clone()
    for s in range(1, S):
        logits += part[s, :, :V]
    if bias is not None:
        logits += bias
    return part.cuda(), (bias.cuda() if bias is not None else None), logits


def _lse(l64):
    m = l64.max(axis=1, keepdims=True)
    return m[:, 0] + np.log(np.exp(l64 - m).sum(axis=1))


_WIDE = [6145, 8192, 8193, 12001, 40000, 65536]


@pytest.mark.parametrize("S", [1, 3, 6])
@pytest.mark.parametrize("V", _WIDE)
def test_split_tail_greedy_and_argmax_against_float64(V, S):
    B, unk = 64, V - 1
    part, bias, logits = _planes(V, S, B, seed=V + S, unk_boost=8.0)      # UNK on top of some rows
    embed = torch.randn(V, E_, generator=_gen(V)).cuda()
    l64 = logits.double().numpy()
    want_tok, want_lp = pick_reference(l64, unk)
    assert (l64.argmax(1) == unk).any()
    o = _PickOut(B, image=True)
    capi.op_reduce_pick_split(part, bias, V, capi.VOCAB_GREEDY, o.it, unk=unk, **o.args(embed))
    o.check("split greedy V=%d S=%d" % (V, S), want_tok, want_lp, embed, 1e-5)
    o = _PickOut(B, image=True)
    lg = torch.full((B, V + 8), float("nan"), device="cuda")
    capi.op_reduce_pick_split(part, bias, V, capi.VOCAB_ARGMAX, o.it, logits_out=lg[:, :V], **o.args(embed))
    tok = l64.argmax(1)
    o.check("split argmax V=%d S=%d" % (V, S), tok, l64[np.arange(B), tok] - _lse(l64), embed, 1e-5)
    assert torch.equal(lg[:, :V].cpu(), logits) and torch.isnan(lg[:, V:]).all()


@pytest.mark.parametrize("tau", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("V", _WIDE)
def test_split_tail_sampling_against_float64(V, S, tau):
    """The draw argmax(l / tau + g) with g the noise of sample_ref.py on every row whose fp64 top-2 key gap exceeds 1e-5, the untempered
    log-probability within 1e-5.  S = 1 without bias is the plain loop path."""
    B, step, seed = 64, 5, 0xC0FFEE + V + S
    part, bias, logits = _planes(V, S, B, seed=3 * V + S, with_bias=S > 1)
    embed = torch.randn(V, E_, generator=_gen(V + 1)).cuda()
    l64 = logits.double().numpy()
    key = l64 / tau + SR.gumbel_noise(seed, np.arange(B), step, V)
    srt = np.sort(key, axis=1)
    rows = np.nonzero(srt[:, -1] - srt[:, -2] > 1e-5)[0]
    assert rows.size >= 0.95 * B
    tok = key.argmax(1)
    o = _PickOut(B, image=True)
    capi.op_reduce_pick_split(part, bias, V, capi.VOCAB_SAMPLE, o.it, temperature=tau, seed=seed, step=step, **o.args(embed))
    o.check("split sample V=%d S=%d tau=%g" % (V, S, tau), tok, l64[np.arange(B), tok] - _lse(l64), embed, 1e-5, rows=rows)


@pytest.mark.parametrize("V", [2, 301, 1025, 4905, 6144])
def test_split_tail_equals_the_register_tails_up_to_6144_words(V):
    B, S = 100, 3
    part, bias, _ = _planes(V, S, B, seed=7 * V)
    embed = torch.randn(V, E_, generator=_gen(V + 2)).cuda()
    a, b = _PickOut(B), _PickOut(B)
    capi.op_reduce_pick(part, bias, V, V - 1, a.it, **a.args(embed))
    capi.op_reduce_pick_split(part, bias, V, capi.VOCAB_GREEDY, b.it, unk=V - 1, **b.args(embed))
    torch.cuda.synchronize()
    assert torch.equal(a.it, b.it) and torch.equal(a.xt, b.xt)
    assert float((a.logp - b.logp)[:, T_].abs().max()) <= 1e-6
    a, b = _PickOut(B), _PickOut(B)
    capi.op_reduce_sample(part, bias, V, 0.7, 1234, 2, a.it, **a.args(embed))
    capi.op_reduce_pick_split(part, bias, V, capi.VOCAB_SAMPLE, b.it, temperature=0.7, seed=1234, step=2, **b.args(embed))
    torch.cuda.synchronize()
    assert torch.equal(a.it, b.it) and torch.equal(a.xt, b.xt)
    assert float((a.logp - b.logp)[:, T_].abs().max()) <= 1e-6


@pytest.mark.parametrize("V,unk", [(6145, 6144), (8193, 0), (9001, 4500), (40000, 39999)])
def test_split_tail_on_tie_and_unk_rows(V, unk):
    """sampler_ref's special rows (ties inside a warp, across warps, 1024 words apart = across slices, UNK on top / tied) as exact sums."""
    B = 60
    x, kinds = special_rows(B, V, unk, seed=V + unk)
    want_tok, want_lp = pick_reference(x, unk)
    planes, bias, _, _ = _exact_operands(x, seed=V)
    embed = torch.randn(V, E_, generator=_gen(V + 3)).cuda()
    o = _PickOut(B, image=True)
    capi.op_reduce_pick_split(planes, bias, V, capi.VOCAB_GREEDY, o.it, unk=unk, **o.args(embed))
    o.check("split special V=%d" % V, want_tok, want_lp, embed, 1e-5, kinds=kinds)


def test_split_tail_nan_rows_and_determinism():
    """All-NaN rows give token 0; repeated launches give bit-identical outputs whichever CTA of a row finishes last."""
    V, B, S = 40000, 100, 4
    part, bias, _ = _planes(V, S, B, seed=11)
    part[:, :3, :V] = float("nan")
    embed = torch.randn(V, E_, generator=_gen(12)).cuda()
    for mode, kw in ((capi.VOCAB_GREEDY, dict(unk=V - 1)), (capi.VOCAB_SAMPLE, dict(temperature=0.9, seed=77, step=3))):
        ref = None
        for _ in range(5):
            o = _PickOut(B, image=True)
            capi.op_reduce_pick_split(part, bias, V, mode, o.it, **kw, **o.args(embed))
            torch.cuda.synchronize()
            got = (o.it.clone(), o.logp.clone(), o.xt.clone(), o.img.clone())
            assert bool((got[0][:3] == 0).all())
            if ref is None:
                ref = got
            assert all(torch.equal(a, b) for a, b in zip(got[:1] + got[2:], ref[:1] + ref[2:]))
            assert torch.equal(torch.nan_to_num(got[1], 1.0), torch.nan_to_num(ref[1], 1.0))


def test_split_tail_rejects_bad_arguments():
    it = torch.zeros(4, dtype=torch.int64, device="cuda")
    with pytest.raises(capi.GvdError):               # pitch not a multiple of 4
        capi.op_reduce_pick_split(torch.zeros(1, 4, 6147, device="cuda"), None, 6145, capi.VOCAB_GREEDY, it)
    with pytest.raises(capi.GvdError):
        capi.op_reduce_pick_split(torch.zeros(1, 4, 6148, device="cuda"), None, 6145, capi.VOCAB_SAMPLE, it, temperature=0.0)
    with pytest.raises(capi.GvdError):
        capi.op_reduce_pick_split(torch.zeros(1, 4, 6148, device="cuda"), None, 6145, 7, it)


# ------------------------------------------------------------------------------------------------------------ model level
def _names(kind):
    return [n for n, c in CASES.items() if c["kind"] == kind]


_models = {}


def _case(name, case=None):
    if name not in _models:
        from gvd_b200.misc.AttModel import TopDownModel
        opt, sd, inp = build_case(case or CASES[name])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m = TopDownModel(opt)
        m.load_state_dict(sd)
        _models[name] = (opt, sd, inp, m.cuda().eval())
    return _models[name]


def _maxerr(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def _greedy(model, inp):
    dev = {k: inp[k].cuda() for k in KEYS}
    with torch.no_grad():
        out = model._sample(*(dev[k] for k in KEYS), {"sample_max": 1, "beam_size": 1})
    torch.cuda.synchronize()
    return tuple(o.cpu() for o in out)


@pytest.mark.parametrize("backend", [923, 3, 0])
@pytest.mark.parametrize("name", _names("greedy"))
def test_wide_vocab_greedy_matches_oracle_and_reference(name, backend):
    capi.set_backend(backend)
    opt, sd, inp, model = _case(name)
    fx = load_fixture(name)
    seq, logp, att2, sim = _greedy(model, inp)
    oseq, ologp, oatt2, osim = O.sample_greedy(sd, opt, inp)
    assert torch.equal(seq, oseq) and np.array_equal(seq.numpy(), fx["seq"])
    assert _maxerr(logp, ologp) <= TOL and np.max(np.abs(logp.numpy() - fx["logp"])) <= TOL
    assert _maxerr(att2, oatt2) <= TOL and _maxerr(sim, osim) <= TOL


@pytest.mark.parametrize("name", _names("greedy"))
def test_wide_vocab_graph_replay_equals_direct_enqueue(name):
    """The captured loop and the kernel-by-kernel enqueue (taken while the stage profiler is on) give bit-identical outputs, and the host
    buffer entry point gives the device path's."""
    capi.set_backend(923)
    opt, sd, inp, model = _case(name)
    a = _greedy(model, inp)
    capi.profile_enable(True)
    b = _greedy(model, inp)
    capi.profile_enable(False)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    pinned = {k: inp[k].pin_memory() for k in KEYS}
    out = model._native.sample_greedy_host(*(pinned[k] for k in KEYS))
    assert torch.equal(out["seq"], a[0]) and torch.equal(out["logp"], a[1])


@pytest.mark.parametrize("backend", [923, 3, 0])
@pytest.mark.parametrize("name", ["v9001_greedy_small_B5", "v40000_greedy_small_B4"])
def test_wide_vocab_multinomial_matches_oracle(name, backend):
    """gvd_decode_sample (refused above 6144 words before the sliced tail) against the oracle's multinomial loop with the same noise; the
    seed is the first whose oracle run has no near-tie (top-2 key gap < 1e-3) at any step."""
    capi.set_backend(backend)
    opt, sd, inp, model = _case(name)
    B, T = inp["segs_feat"].shape[:2]
    tau = 0.8
    feats = O.prologue(sd, opt, *(inp[k] for k in KEYS))
    for seed in range(1, 40):
        oseq, ologp, oatt2, _, gaps = SR.sample_multinomial(sd, opt, inp, tau, SR.noise_fn(seed, np.arange(B), opt.vocab_size), feats=feats)
        if (gaps >= 1e-3).all():
            break
    else:
        pytest.fail("no seed without a near-tie")
    nm = model._native_model()
    dev = {k: inp[k].cuda() for k in KEYS}
    nm.prologue(*(dev[k] for k in KEYS))
    seq, logp, att2 = (o.cpu() for o in nm.decode_sample(B, T, dev["pnt_mask"], seed, tau))
    torch.cuda.synchronize()
    assert torch.equal(seq, oseq)
    assert _maxerr(logp, ologp) <= TOL and _maxerr(att2, oatt2) <= TOL


@pytest.mark.parametrize("backend", [923, 3, 0])
@pytest.mark.parametrize("name", _names("beam"))
def test_wide_vocab_beam_matches_reference(name, backend):
    capi.set_backend(backend)
    case = CASES[name]
    opt, sd, inp, model = _case(name)
    fx = load_fixture(name)
    dev = {k: inp[k].cuda() for k in KEYS}
    with torch.no_grad():
        seq, logp, att, _ = model._sample(*(dev[k] for k in KEYS), {"beam_size": case["beam_size"]})
    torch.cuda.synchronize()
    assert np.array_equal(seq.cpu().numpy(), fx["seq"]) and np.array_equal(att.cpu().numpy(), fx["att2_idx"])
    assert np.max(np.abs(logp.cpu().numpy() - fx["logp"])) <= TOL


def _teacher(model, inp, mode):
    dev = {k: v.cuda() for k, v in inp.items()}
    with torch.no_grad():
        out = model(dev["segs_feat"], dev["input_seq"], dev["gt_seq"], dev["num"], dev["ppls"], dev["gt_boxes"], dev["mask_boxes"],
                    dev["ppls_feat"], dev["frm_mask"], dev["sample_idx"], dev["pnt_mask"], mode)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("backend", [923, 3, 0])
def test_wide_vocab_mle_and_grd_match_reference(backend):
    capi.set_backend(backend)
    opt, sd, inp, model = _case("v9001_mle_small_B5")
    got = np.array([float(l) for l in _teacher(model, inp, "MLE")])
    assert np.max(np.abs(got - load_fixture("v9001_mle_small_B5")["losses"])) <= TOL
    opt, sd, inp, model = _case("v9001_grd_small_B5")
    fx = load_fixture("v9001_grd_small_B5")
    cls_pred, att_idx, grd_idx = _teacher(model, inp, "GRD")
    assert np.array_equal(cls_pred.cpu().numpy(), fx["cls_pred"])
    assert np.array_equal(att_idx.cpu().numpy(), fx["att_idx"]) and np.array_equal(grd_idx.cpu().numpy(), fx["grd_idx"])


def test_wide_vocab_training_step_against_oracle():
    from gvd_b200.train import TrainStep
    from gvd_b200.train_ops import NativeOps
    opt, sd, inp = build_case(CASES["v9001_mle_small_B5"])
    losses, loss, grads, total_norm, new = O.train_step(sd, opt, inp)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    l2, loss2, g2, tn2, new2 = TrainStep(NativeOps()).step({k: v.cuda() for k, v in sd.items()}, opt, dev, host=inp)
    torch.cuda.synchronize()
    assert abs(float(loss2.cpu()) - float(loss)) <= TOL
    for a, b in zip(losses, l2):
        assert abs(float(a) - float(b.cpu())) <= TOL
    assert sorted(g2.keys()) == sorted(grads.keys())
    scale = float(total_norm)
    assert abs(tn2 - scale) <= 1e-4 * scale
    for k in grads:
        a, b = grads[k], g2[k].cpu().reshape(grads[k].shape)
        assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()) + 1e-6 * scale, k


@pytest.mark.parametrize("backend", [923, 3, 0])
def test_wide_vocab_transformer_greedy(backend):
    """Above 12000 words the transformer head runs the sliced tail in its argmax mode: predictions, the logits of every step and the
    teacher-forced loss against the oracle and the fixture."""
    capi.set_backend(backend)
    name = "v13001_tfm_greedy_small_B4"
    opt, sd, inp, model = _case(name)
    fx = load_fixture(name)
    dev = {k: v.cuda() for k, v in inp.items()}
    d = torch.zeros(inp["ppls"].shape[0], dtype=torch.uint8, device="cuda")
    with torch.no_grad():
        seq = model(dev["segs_feat"], d, d, dev["num"], dev["ppls"], d, d, dev["ppls_feat"], d, dev["sample_idx"], dev["pnt_mask"], "sample",
                    {"sample_max": 1, "beam_size": 1})[0]
    torch.cuda.synchronize()
    oseq, _, _, trace = O.tfm_sample(sd, opt, inp, return_trace=True)
    assert torch.equal(seq.cpu(), oseq) and np.array_equal(seq.cpu().numpy(), fx["seq"])
    B, T = inp["segs_feat"].shape[:2]
    nm = model._native_model()
    seq2, logits = model._tfm.decode_greedy(*model._tfm_encodings(nm, B, T), want_logits=True)
    torch.cuda.synchronize()
    assert torch.equal(seq2, seq)
    assert float((logits.cpu().double() - torch.stack(trace, 1).double()).abs().max()) <= TOL
    assert float(np.abs(subsample("tfm_logits", logits.cpu()).numpy().astype(np.float64) - fx["tfm_logits"]).max()) <= TOL
    # teacher forcing through the same tail: the loss against the oracle
    opt2, sd2, inp2 = build_case(dict(CASES[name], kind="tfm_mle"))
    dev2 = {k: v.cuda() for k, v in inp2.items()}
    with torch.no_grad():
        out = model(dev2["segs_feat"], dev2["input_seq"], dev2["gt_seq"], dev2["num"], dev2["ppls"], dev2["gt_boxes"], dev2["mask_boxes"],
                    dev2["ppls_feat"], dev2["frm_mask"], dev2["sample_idx"], dev2["pnt_mask"], "MLE")
    torch.cuda.synchronize()
    assert abs(float(out[0]) - float(O.tfm_mle(sd2, opt2, inp2))) <= TOL


@pytest.mark.parametrize("V", [8192, 32000])
def test_full_size_greedy_and_sampling(V):
    """B = 100, T = 10 at the full model dims (fp16x3 split-K products): greedy and multinomial decoding of 100 clips, the first 16 against
    the oracle (run on the device) wherever its decision margin exceeds 1e-4 at every step.  8192 words: split-K head + sliced tail;
    32000 words: no split plan, the generic head GEMM + sliced tail on one plane (which also writes the fp16x3 image of the next input)."""
    capi.set_backend(923)
    case = dict(kind="greedy", B=100, opt=dict(t_attn_size=10, vocab_size=V), input_seed=321)
    opt, sd, inp, model = _case("full_v%d" % V, case)
    seq, logp, att2, sim = _greedy(model, inp)
    n = 16
    sub = {k: v[:n].cuda() for k, v in inp.items()}
    sdc = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        oseq, ologp, oatt2, _, trace = O.sample_greedy(sdc, opt, sub, return_trace=True)
    lp = torch.stack([t["logprobs"] for t in trace], 1).cpu()                  # [n, L, V]
    top = torch.topk(lp, 3, dim=-1).values
    unk = int(opt.wtoi["UNK"])
    top1 = lp.argmax(-1)
    margin = torch.where(top1 == unk, top[..., 1] - top[..., 2], top[..., 0] - top[..., 1]).min(1).values
    rows = torch.nonzero(margin > 1e-4).flatten()
    assert rows.numel() >= n // 2, margin
    assert torch.equal(seq[rows], oseq.cpu()[rows])
    assert _maxerr(logp[rows], ologp.cpu()[rows]) <= TOL and _maxerr(att2[rows], oatt2.cpu()[rows]) <= TOL
    nm = model._native_model()
    B, T = inp["segs_feat"].shape[:2]
    dev = {k: inp[k].cuda() for k in KEYS}
    nm.prologue(*(dev[k] for k in KEYS))
    s1 = nm.decode_sample(B, T, dev["pnt_mask"], 5, 1.0)[0].clone()
    s2 = nm.decode_sample(B, T, dev["pnt_mask"], 5, 1.0)[0]
    torch.cuda.synchronize()
    assert torch.equal(s1, s2) and int(s1.min()) >= 0 and int(s1.max()) < opt.vocab_size
    assert not torch.equal(s1, seq.cuda())
