"""region_attn_mode 'dp' and 'mix_mul' of the top-down captioner on the device: the decode attention op by op against float64 in every form,
and every decode / training entry point against the oracle's step of the mode (tests/region_attn_oracle.py) and the reference's fixtures
(tests/golden/region_attn_cases.py).  Bars as tests/test_gpu_parity.py: token ids and argmax indices bit-exact, attention logits / log-probs /
losses within 1e-4 (the dp logits, unscaled A-wide dot products, within 1e-4 of their magnitude)."""
import warnings

import numpy as np
import pytest
import torch

import sample_ref as SR
from cases import CASES as BASE_CASES, build_case, load_fixture
from gvd_b200 import capi
from region_attn_cases import REGION_ATTN_CASES as CASES
from region_attn_oracle import RegionAttnRefOps, oracle_modes
from test_gpu_attn_beam_ops import EPS32, MIN_VALUE, NAN, TANH_ERR, _Attn, _chunk_ref, _gen

pytestmark = pytest.mark.gpu
TOL = 1e-4
KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


@pytest.fixture(autouse=True)
def _restore_backend():
    b = capi.get_backend()
    yield
    capi.set_backend(b)


def _maxerr(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def _names(kind):
    return [n for n, c in CASES.items() if c["kind"] == kind]


def _ztol(fx_att2):
    """The logit bar: 1e-4, relative for the dp logits (A-wide dot products of magnitude up to ~10)."""
    live = np.abs(fx_att2[fx_att2 > -1e7])
    return TOL * max(1.0, float(live.max()) if live.size else 1.0)


_models = {}


def _case(name):
    """(opt, state_dict, inputs, module in eval mode), the module built once per case."""
    if name not in _models:
        from gvd_b200.misc.AttModel import TopDownModel
        opt, sd, inp = build_case(CASES[name])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m = TopDownModel(opt)
        m.load_state_dict(sd)
        _models[name] = (opt, sd, inp, m.cuda().eval())
    return _models[name]


# ------------------------------------------------------------------------------------------------------------ the decode attention, op by op
def _scores(form, p, q, w, b):
    """fp64 Attention2 score (AttModel.py:79-96) of rows p [B, N, A] against q [B, A]."""
    if form == "dp":
        return torch.einsum("bna,ba->bn", p, q)
    return torch.tanh(p * q[:, None] if form == "mix_mul" else p + q[:, None]) @ w + b


def _bar(form, p, q, w):
    """Error bar of one region logit from the fp32 accumulation: each lane chains A/32 fmaf terms, then a 5-level warp tree and the bias.
    mix / mix_mul: the tanh_mufu error and the rounding of p + q (p q) through tanh (slope <= 1), times ||w||_1, plus the sum's rounding.
    dp: no tanh, so the sum's rounding alone, (A/32 + 8) eps32 times the largest sum of |p_a q_a| of a row."""
    A = p.shape[-1]
    if form == "dp":
        return EPS32 * (A / 32 + 8) * float(torch.einsum("bna,ba->bn", p.abs(), q.abs()).max())
    pmax, qmax = float(p.abs().max()), float(q.abs().max())
    pq = pmax * qmax if form == "mix_mul" else pmax + qmax
    return float(w.abs().sum()) * (TANH_ERR + EPS32 * (pq + A / 32 + 8))


def _problem(B, R, T, A, H, RC, TC, div, seed):
    P = _Attn(B, R, T, A, H, RC, TC, div, seed=seed, mask_stride=True)
    g = _gen(seed + 7)
    P.gate_w = (torch.randn(H, generator=g) * 3 / H ** 0.5).cuda()
    P.gate_b = (torch.randn(1, generator=g) * 0.3).cuda()
    hbuf = torch.full((B, H + 8), NAN)
    hbuf[:, 4:4 + H] = torch.tanh(torch.randn(B, H, generator=g))
    P.gate_h = hbuf.cuda()[:, 4:4 + H]
    return P


def _run(P, form, mode, q=None, q_part=None, q_bias=None, fused=True, x_ld=None, image=False):
    """One launch of gvd_op_attention_form; in 'dp' the region alpha_net pointers are NULL."""
    B, R, H = P.B, P.R, P.H
    dual = mode == "dual_region"
    zbuf = torch.full((B, R + 5), NAN, device="cuda")
    xbuf = torch.full((B, x_ld or H), NAN, device="cuda")
    x = xbuf[:, H:2 * H] if x_ld else xbuf
    part = torch.full((B, 2 * P.nch_r if dual else P.nch_r + P.nch_t, H + 4), NAN, device="cuda")
    ticket = torch.zeros(B, dtype=torch.int32, device="cuda") if fused else None
    Hp = (H + 31) // 32 * 32
    img = torch.full((B, 2 * Hp), -1, dtype=torch.int32, device="cuda") if image else None
    if q is None and q_part is None:
        q = P.q
    dp = form == "dp"
    w1, b1 = (None, None) if dp and dual else (P.w1, P.b1)
    w2, b2 = (None, None) if dp else (P.w2, P.b2)
    capi.op_attention(P.p_pool, None if mode == "featmap" else P.pool, None if dual else P.p_conv, None if dual else P.conv, w1, b1, w2, b2,
                      P.att_mask, P.out_mask, zbuf[:, :R], part, x, P.RC, P.TC, q=q, q_part=q_part, q_bias=q_bias, ticket=ticket,
                      x_pk=img[:, :Hp] if image else None, feat_div=P.div, att_input_mode=mode,
                      gate_w=P.gate_w if dual else None, gate_b=P.gate_b if dual else None, gate_h=P.gate_h if dual else None,
                      region_attn_mode=form)
    torch.cuda.synchronize()
    return zbuf, x, xbuf, part, ticket, img


def _check(P, form, mode, zbuf, x, xbuf, part, img=None, q=None):
    """fp64: the masked logits z_out, the chunk records of every region attention (and the temporal ones), and x."""
    A, R, H = P.A, P.R, P.H
    d = lambda t: t.double()
    idx = torch.arange(P.B, device="cuda") // P.div
    q = d(P.q if q is None else q)
    pp, pool = d(P.p_pool)[idx], d(P.pool)[idx]
    am = P.att_mask[idx][:, 1:].bool()
    dual = mode == "dual_region"
    z = _scores(form, pp, q[:, A:], d(P.w2), d(P.b2)).masked_fill(am, MIN_VALUE)
    bar = _bar(form, pp, q[:, A:], d(P.w2))
    branches = [(z, bar, 0)]                                            # the region chunks' records come first
    att2 = torch.einsum("br,brh->bh", torch.softmax(z, 1), pool)
    if dual:
        zd = _scores(form, pp, q[:, :A], d(P.w1), d(P.b1)).masked_fill(am, MIN_VALUE)
        bar_d = _bar(form, pp, q[:, :A], d(P.w1))
        branches = [(z, bar, 0), (zd, bar_d, P.nch_r)]
        g = torch.sigmoid(d(P.gate_h) @ d(P.gate_w) + d(P.gate_b))[:, None]
        x_ref = g * att2 + (1 - g) * torch.einsum("br,brh->bh", torch.softmax(zd, 1), pool)
        bars = [bar, bar_d]
    else:
        conv = d(P.conv)[idx]
        s = torch.tanh(d(P.p_conv)[idx] + q[:, None, :A]) @ d(P.w1) + d(P.b1)
        bar_t = _bar("mix", d(P.p_conv)[idx], q[:, :A], d(P.w1))
        att = torch.einsum("bt,bth->bh", torch.softmax(s, 1), conv)
        x_ref = att if mode == "featmap" else att + att2
        bars = [bar_t] + ([] if mode == "featmap" else [bar])
        m, l, _ = _chunk_ref(s, conv, P.TC)
        tmp = part[:, P.nch_r:].double()
        assert float((tmp[..., 0] - m).abs().max()) <= bar_t
    z_out = z.masked_fill(P.out_mask[idx][:, 1:].bool(), MIN_VALUE)
    zz = zbuf[:, :R]
    masked = z_out == MIN_VALUE
    assert torch.equal(zz.double()[masked], z_out[masked])
    if (~masked).any():
        assert float((zz.double() - z_out)[~masked].abs().max()) <= bar, (float((zz.double() - z_out)[~masked].abs().max()), bar)
    assert torch.isnan(zbuf[:, R:]).all()
    for sc, bb, c0 in branches:
        m, l, acc = _chunk_ref(sc, pool, P.RC)
        got = part[:, c0:c0 + P.nch_r].double()
        assert float((got[..., 0] - m).abs().max()) <= bb
        assert float(((got[..., 1] - l) / l).abs().max()) <= 2 * bb + 1e-6 * P.RC
        if mode == "featmap":
            assert bool(torch.isnan(got[..., 4:]).all())              # featmap: the region chunks store no weighted sum
        else:
            assert float(((got[..., 4:] - acc).abs() / (l[..., None] * float(pool.abs().max()))).max()) <= 2 * bb + 1e-6 * P.RC
    fmax = float(pool.abs().max()) if dual else max(float(pool.abs().max()), float(d(P.conv).abs().max()))
    err = float((x.double() - x_ref).abs().max()) / fmax
    assert err <= 2 * sum(bars) + 1e-5, (err, bars)
    if xbuf.shape[1] > H:
        assert torch.isnan(xbuf[:, :H]).all() and torch.isnan(xbuf[:, 2 * H:]).all()
    if img is not None:
        from test_gpu_tcgen05 import _decode_f16x3
        Hp = (H + 31) // 32 * 32
        val, _ = _decode_f16x3(img[:, :Hp].contiguous(), H, 4.0)
        xv = x.cpu().double().numpy()
        assert float(np.abs(val - xv).max()) <= 2.0 ** -20 * max(1.0, float(np.abs(xv).max()))
    return err, bar


_FORM_CASES = [   # B, R, T, A, H, RC, TC, feat_div: the decode attention's shapes (A = 96 generic, 128 .. 512 the register paths AJ = 1 .. 4)
    (5, 52, 10, 96, 248, 16, 16, 1),
    (5, 52, 10, 512, 248, 7, 7, 1),
    (3, 129, 480, 512, 1024, 80, 128, 1),
    (100, 1000, 10, 512, 1024, 128, 16, 1),
    (12, 52, 10, 512, 1024, 16, 16, 3),
    (128, 13, 10, 256, 248, 7, 16, 4),
    (6, 40, 12, 128, 248, 16, 16, 2),
    (4, 100, 10, 384, 512, 32, 16, 1),
]


@pytest.mark.parametrize("mode", ["both", "featmap", "dual_region"])
@pytest.mark.parametrize("form", ["mix_mul", "dp"])
@pytest.mark.parametrize("B,R,T,A,H,RC,TC,div", _FORM_CASES, ids=["B%d-R%d-T%d-A%d-H%d-RC%d-TC%d-div%d" % c for c in _FORM_CASES])
def test_region_attention_form_against_fp64(B, R, T, A, H, RC, TC, div, form, mode):
    """gvd_op_attention_form: fused merge into a column window with its fp16x3 image against fp64; the separate combine kernel is bit-equal
    to the fused merge (dual_region has the fused merge only: a relaunch is bit-equal); the tickets are left at zero."""
    P = _problem(B, R, T, A, H, RC, TC, div, seed=B * 7 + R + T + A + H + RC + TC + div)
    zbuf, x, xbuf, part, ticket, img = _run(P, form, mode, x_ld=3 * H, image=True)
    err, bar = _check(P, form, mode, zbuf, x, xbuf, part, img)
    print("%s/%s attention B=%d R=%d T=%d A=%d H=%d RC=%d div=%d: |x err|/max|f| %.2e, logit bar %.2e" % (form, mode, B, R, T, A, H, RC, div,
                                                                                                       err, bar))
    assert bool((ticket == 0).all())
    zbuf2, x2, _, _, _, _ = _run(P, form, mode, fused=mode == "dual_region")
    assert torch.equal(zbuf2[:, :R], zbuf[:, :R]) and torch.equal(x2, x)


@pytest.mark.parametrize("mode", ["both", "dual_region"])
@pytest.mark.parametrize("form", ["mix_mul", "dp"])
@pytest.mark.parametrize("q_S", [1, 3, 4])
def test_region_attention_form_query_from_split_k_planes(q_S, form, mode):
    B, R, T, A, H = 7, 52, 10, 512, 1024
    P = _problem(B, R, T, A, H, 16, 16, 1, seed=80 + q_S)
    g = _gen(400 + q_S)
    q_part = (torch.randn(q_S, B, 2 * A, generator=g) * 0.3).cuda()
    q_bias = (torch.randn(2 * A, generator=g) * 0.3).cuda()
    q = q_bias.expand(B, 2 * A).clone()
    for s in range(q_S):
        q += q_part[s]
    zbuf, x, xbuf, part, _, _ = _run(P, form, mode, q_part=q_part, q_bias=q_bias, x_ld=3 * H)
    zbuf_d, x_d, _, _, _, _ = _run(P, form, mode, q=q)
    assert torch.equal(zbuf[:, :R], zbuf_d[:, :R]) and torch.equal(x, x_d)
    _check(P, form, mode, zbuf, x, xbuf, part, q=q)


@pytest.mark.parametrize("mode", ["both", "featmap", "dual_region"])
def test_region_attention_mix_form_is_the_mode_entry_point(mode):
    """gvd_op_attention_form('mix') and gvd_op_attention_mode are the same launch: bit-equal outputs."""
    P = _problem(12, 52, 10, 512, 1024, 16, 16, 3, seed=5)
    a = _run(P, "mix", mode, x_ld=3 * 1024)
    dual = mode == "dual_region"
    zbuf = torch.full((12, 57), NAN, device="cuda")
    xbuf = torch.full((12, 3 * 1024), NAN, device="cuda")
    part = torch.full(tuple(a[3].shape), NAN, device="cuda")
    capi.op_attention(P.p_pool, None if mode == "featmap" else P.pool, None if dual else P.p_conv, None if dual else P.conv, P.w1, P.b1, P.w2,
                      P.b2, P.att_mask, P.out_mask, zbuf[:, :52], part, xbuf[:, 1024:2048], 16, 16, q=P.q,
                      ticket=torch.zeros(12, dtype=torch.int32, device="cuda"), feat_div=3, att_input_mode=mode,
                      gate_w=P.gate_w if dual else None, gate_b=P.gate_b if dual else None, gate_h=P.gate_h if dual else None)
    torch.cuda.synchronize()
    assert torch.equal(zbuf[:, :52], a[0][:, :52]) and torch.equal(xbuf[:, 1024:2048], a[1])


def test_region_attention_form_rejects_missing_weights():
    """mix_mul reads the region alpha_net, so NULL is refused (dp is the only form that runs without it)."""
    P = _problem(3, 13, 4, 96, 248, 7, 7, 1, seed=1)
    with pytest.raises(capi.GvdError):
        capi.op_attention(P.p_pool, P.pool, P.p_conv, P.conv, P.w1, P.b1, None, None, P.att_mask, P.out_mask, torch.empty(3, 13, device="cuda"),
                          torch.empty(3, 3, 252, device="cuda"), torch.empty(3, 248, device="cuda"), 7, 7, q=P.q, region_attn_mode="mix_mul")


# ------------------------------------------------------------------------------------------------------------ decode entry points
def _greedy(model, inp):
    dev = {k: inp[k].cuda() for k in KEYS}
    with torch.no_grad():
        seq, logp, att2, sim = model._sample(*(dev[k] for k in KEYS), {"sample_max": 1, "beam_size": 1})
    torch.cuda.synchronize()
    return seq.cpu(), logp.cpu(), att2.cpu(), sim.cpu()


@pytest.mark.parametrize("backend", [923, 3, 0])
@pytest.mark.parametrize("name", _names("greedy"))
def test_region_attn_greedy_matches_oracle_and_reference(name, backend):
    """The three product paths of the step (923: split-K fp16x3 products, 3: tensor-core products, 0: CUDA-core products)."""
    capi.set_backend(backend)
    opt, sd, inp, model = _case(name)
    fx = load_fixture(name)
    seq, logp, att2, sim = _greedy(model, inp)
    with oracle_modes(opt) as O:
        oseq, ologp, oatt2, osim = O.sample_greedy(sd, opt, inp)
    ztol = _ztol(fx["att2"])
    assert torch.equal(seq, oseq) and np.array_equal(seq.numpy(), fx["seq"])
    assert _maxerr(logp, ologp) <= TOL and np.max(np.abs(logp.numpy() - fx["logp"])) <= TOL
    assert _maxerr(att2, oatt2) <= ztol and np.max(np.abs(att2.numpy() - fx["att2"])) <= ztol
    assert torch.equal(att2 == -1e8, oatt2 == -1e8)
    assert _maxerr(sim, osim) <= TOL


@pytest.mark.parametrize("name", ["dp_greedy_small_B5", "mul_greedy_small_B5", "dp_dual_greedy_small_B5"])
def test_region_attn_host_buffer_entry_point_matches_device_path(name):
    opt, sd, inp, model = _case(name)
    seq, logp, att2, sim = _greedy(model, inp)
    pinned = {k: inp[k].pin_memory() for k in KEYS}
    out = model._native.sample_greedy_host(*(pinned[k] for k in KEYS))
    assert torch.equal(out["seq"], seq) and torch.equal(out["logp"], logp) and torch.equal(out["att2"], att2) and torch.equal(out["sim"], sim)


@pytest.mark.parametrize("name", ["dp_greedy_small_B5", "mul_greedy_small_B5", "dp_featmap_greedy_small_B5", "dp_dual_greedy_small_B5",
                                  "mul_dual_greedy_small_B5"])
def test_region_attn_decode_step_matches_oracle_step(name):
    """gvd_decode_step_fwd: one teacher-fed step at a time, h_lang and the masked logits against the oracle's step of the mode."""
    opt, sd, inp, model = _case(name)
    B, T = inp["segs_feat"].shape[:2]
    nm = model._native_model()
    dev = {k: inp[k].cuda() for k in KEYS}
    nm.prologue(*(dev[k] for k in KEYS))
    nm.reset_state(B, T)
    with oracle_modes(opt) as O:
        feats = O.prologue(sd, opt, *(inp[k] for k in KEYS))
        H = opt.rnn_size
        state = (torch.zeros(2, B, H), torch.zeros(2, B, H))
        g = _gen(9)
        for t in range(4):
            tok = torch.randint(1, opt.vocab_size, (B,), generator=g)
            z = torch.empty(B, nm.R, device="cuda")
            h = torch.empty(B, H, device="cuda")
            nm.decode_step(B, T, t, tok.cuda(), dev["pnt_mask"], dev["pnt_mask"], z, nm.R, h)
            torch.cuda.synchronize()
            oh, state, oz, _ = O.core_step(sd, O.embed_tokens(sd, tok), feats, inp["pnt_mask"], inp["pnt_mask"], state)
            assert _maxerr(h, oh) <= TOL and _maxerr(z, oz) <= TOL * max(1.0, float(oz[oz > -1e7].abs().max())), t


@pytest.mark.parametrize("backend", [923, 0])
@pytest.mark.parametrize("name", ["dp_greedy_small_B5", "dp_greedy_T10_B3", "mul_greedy_small_B5", "mul_greedy_T10_B3"])
def test_region_attn_multinomial_matches_oracle(name, backend):
    """gvd_decode_sample against the oracle's multinomial loop with the same counter-based noise; the seed is the first whose oracle run has
    no near-tie (top-2 key gap < 1e-3) at any step."""
    capi.set_backend(backend)
    opt, sd, inp, model = _case(name)
    B, T = inp["segs_feat"].shape[:2]
    rows = np.arange(B)
    tau = 0.8
    with oracle_modes(opt) as O:
        feats = O.prologue(sd, opt, *(inp[k] for k in KEYS))
        for seed in range(1, 40):
            oseq, ologp, oatt2, _, gaps = SR.sample_multinomial(sd, opt, inp, tau, SR.noise_fn(seed, rows, opt.vocab_size), feats=feats)
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
    assert _maxerr(logp, ologp) <= TOL and _maxerr(att2, oatt2) <= TOL * max(1.0, float(oatt2[oatt2 > -1e7].abs().max()))


@pytest.mark.parametrize("name", _names("beam"))
def test_region_attn_beam_matches_oracle_and_reference(name):
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


@pytest.mark.parametrize("name", _names("mle"))
def test_region_attn_mle_losses_match_reference(name):
    opt, sd, inp, model = _case(name)
    got = np.array([float(l) for l in _teacher(model, inp, "MLE")])
    assert np.max(np.abs(got - load_fixture(name)["losses"])) <= TOL


@pytest.mark.parametrize("name", _names("grd"))
def test_region_attn_grd_indices_match_reference(name):
    opt, sd, inp, model = _case(name)
    fx = load_fixture(name)
    cls_pred, att_idx, grd_idx = _teacher(model, inp, "GRD")
    assert np.array_equal(cls_pred.cpu().numpy(), fx["cls_pred"])
    assert np.array_equal(att_idx.cpu().numpy(), fx["att_idx"]) and np.array_equal(grd_idx.cpu().numpy(), fx["grd_idx"])


def test_transformer_loads_a_dp_checkpoint():
    """att_model='transformer' with region_attn_mode 'dp': the state_dict lacks core.attention2.alpha_net.* and the decode, which never runs
    the region attention, is bit-identical to the 'mix' model's on the same tensors."""
    from gvd_b200.misc.AttModel import TopDownModel
    case = BASE_CASES["tfm_greedy_small_B5"]
    outs = []
    for form in ("mix", "dp"):
        opt, sd, inp = build_case(dict(case, opt=dict(case["opt"], region_attn_mode=form)))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m = TopDownModel(opt)
        m.load_state_dict(sd, strict=True)
        m.cuda().eval()
        assert ("core.attention2.alpha_net.weight" in sd) == (form == "mix")
        dev = {k: v.cuda() for k, v in inp.items()}
        d = torch.zeros(inp["ppls"].shape[0], dtype=torch.uint8, device="cuda")
        with torch.no_grad():
            seq = m(dev["segs_feat"], d, d, dev["num"], dev["ppls"], d, d, dev["ppls_feat"], d, dev["sample_idx"], dev["pnt_mask"], "sample",
                    {"sample_max": 1, "beam_size": 1})[0]
        torch.cuda.synchronize()
        outs.append(seq.cpu())
    assert torch.equal(outs[0], outs[1]) and np.array_equal(outs[1].numpy(), load_fixture("tfm_greedy_small_B5")["seq"])


# ------------------------------------------------------------------------------------------------------------ training
@pytest.mark.parametrize("shape", [(5, 52, 96), (3, 1000, 512), (4, 13, 250)])
def test_att_scores_mul_primitives_against_fp64(shape):
    """NativeOps.att_scores_mul / _bwd against float64 autograd of s = w . tanh(p q) + b; the backward is deterministic (bit-equal on a
    rerun)."""
    from gvd_b200.train_ops import NativeOps
    B, N, A = shape
    g = _gen(B + N + A)
    p, q = torch.randn(B, N, A, generator=g) * 0.7, torch.randn(B, A, generator=g) * 0.7
    w, b, ds = torch.randn(1, A, generator=g) / A ** 0.5, torch.randn(1, generator=g), torch.randn(B, N, generator=g)
    ops = NativeOps()
    s = ops.att_scores_mul(p.cuda(), q.cuda(), w.cuda(), b.cuda())
    got = ops.att_scores_mul_bwd(ds.cuda(), p.cuda(), q.cuda(), w.cuda())
    again = ops.att_scores_mul_bwd(ds.cuda(), p.cuda(), q.cuda(), w.cuda())
    torch.cuda.synchronize()
    pd, qd, wd, bd = (t.double().requires_grad_() for t in (p, q, w.reshape(-1), b))
    sd_ = torch.tanh(pd * qd[:, None]) @ wd + bd
    (sd_ * ds.double()).sum().backward()
    # fp32: tanhf and the A-term sums (the forward's warp sum, the colsum kernel's N- and B*N-term sums)
    bar_s = float(w.abs().sum()) * 4 * EPS32 * (1 + A / 32 + 8 + float((p * q[:, None]).abs().max()))
    assert _maxerr(s, sd_.detach()) <= bar_s
    scale = float(ds.abs().max()) * float(w.abs().max())
    for t, ref, n in zip(got, (pd.grad, qd.grad, wd.grad, bd.grad), (1, N, B * N, B * N)):
        assert _maxerr(t.reshape(ref.shape), ref) <= 8 * EPS32 * n * scale * max(1.0, float(p.abs().max()) * float(q.abs().max())) + 1e-6
    assert all(torch.equal(a, b) for a, b in zip(got, again))


@pytest.mark.parametrize("name", _names("train"))
def test_region_attn_training_step_against_oracle(name):
    from gvd_b200.train import TrainStep
    from gvd_b200.train_ops import NativeOps
    opt, sd, inp = build_case(CASES[name])
    with oracle_modes(opt) as O:
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


@pytest.mark.parametrize("name", _names("train"))
def test_region_attn_trainer_two_steps(name):
    """Trainer over NativeOps for two steps against the same Trainer over the torch mock; the tensors without a gradient come out
    bit-identical."""
    from gvd_b200.train import Trainer
    from gvd_b200.train_ops import NativeOps
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    a, b = Trainer(NativeOps(), sd, opt), Trainer(RegionAttnRefOps(), sd, opt)
    for it in range(2):
        la, lossa = a.step(dev, host=inp)
        lb, lossb = b.step(inp)
        torch.cuda.synchronize()
        assert abs(float(lossa.cpu()) - float(lossb)) <= 1e-4 * (1 + 9 * it), it
        for k in a.keys:
            assert float((a.weights[k].cpu() - b.weights[k]).abs().max()) <= 2 * 5e-4 * (it + 1), (it, k)
    no_grad = set(str(k) for k in fx["no_grad_keys"])
    assert set(a.idle) == no_grad
    for k in no_grad:
        assert torch.equal(a.weights[k].cpu(), sd[k]), k


@pytest.mark.parametrize("name", ["dp_train_small_B5", "mul_train_small_B5"])
def test_region_attn_module_train_mode_through_the_driver_contract(name):
    """model.train(); losses = model(..., 'MLE'); loss.backward(): every .grad against the oracle, and no alpha_net parameter in 'dp'."""
    opt, sd, inp = build_case(CASES[name])
    with oracle_modes(opt) as O:
        _, _, grads, total_norm, _ = O.train_step(sd, opt, inp)
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = TopDownModel(opt)
    model.load_state_dict(sd)
    model.cuda().train()
    model.train_dropout = False
    dev = {k: v.cuda() for k, v in inp.items()}
    lm, att2, grd, cls = model(dev["segs_feat"], dev["input_seq"], dev["gt_seq"], dev["num"], dev["ppls"], dev["gt_boxes"], dev["mask_boxes"],
                               dev["ppls_feat"], dev["frm_mask"], dev["sample_idx"], dev["pnt_mask"], "MLE")
    loss = (lm.sum() + opt.w_att2 * att2.sum() + opt.w_grd * grd.sum() + opt.w_cls * cls.sum()) / lm.numel()
    loss.backward()
    torch.cuda.synchronize()
    scale = float(total_norm)
    names = [k for k, _ in model.named_parameters()]
    assert ("core.attention2.alpha_net.weight" in names) == (opt.region_attn_mode != "dp")
    for k, p in model.named_parameters():
        if k in grads:
            assert float((p.grad.cpu() - grads[k]).abs().max()) <= 1e-4 * float(grads[k].abs().max()) + 1e-6 * scale, k
        else:
            assert p.grad is None, k
