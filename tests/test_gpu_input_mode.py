"""att_input_mode 'featmap' and 'dual_region' of the top-down captioner on the device: the decode attention op by op against float64, and every decode / training
entry point against the oracle's step of the mode (tests/input_mode_oracle.py) and the reference's fixtures (tests/golden/input_mode_cases.py).
Bars as tests/test_gpu_parity.py: token ids and argmax indices bit-exact, attention logits / log-probs / losses within 1e-4."""
import warnings

import numpy as np
import pytest
import torch

import sample_ref as SR
from cases import build_case, load_fixture
from gvd_b200 import capi
from input_mode_cases import INPUT_MODE_CASES as CASES
from input_mode_oracle import oracle_mode
from test_gpu_attn_beam_ops import MIN_VALUE, NAN, _Attn, _chunk_ref, _gen

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
def _run_featmap(P, q=None, q_part=None, q_bias=None, fused=True, x_ld=None, image=False):
    B, R, H = P.B, P.R, P.H
    zbuf = torch.full((B, R + 5), NAN, device="cuda")
    xbuf = torch.full((B, x_ld or H), NAN, device="cuda")
    x = xbuf[:, H:2 * H] if x_ld else xbuf
    part = torch.full((B, P.nch_r + P.nch_t, H + 4), NAN, device="cuda")
    ticket = torch.zeros(B, dtype=torch.int32, device="cuda") if fused else None
    img = torch.full((B, 2 * ((H + 31) // 32 * 32)), -1, dtype=torch.int32, device="cuda") if image else None
    if q is None and q_part is None:
        q = P.q
    capi.op_attention(P.p_pool, None, P.p_conv, P.conv, P.w1, P.b1, P.w2, P.b2, P.att_mask, P.out_mask, zbuf[:, :R], part, x, P.RC, P.TC,
                      q=q, q_part=q_part, q_bias=q_bias, ticket=ticket, x_pk=img[:, :(H + 31) // 32 * 32] if image else None,
                      feat_div=P.div, att_input_mode="featmap")
    torch.cuda.synchronize()
    return zbuf, x, xbuf, part, ticket


def _check_featmap(P, zbuf, x, xbuf, part, q=None):
    """featmap: z_out as in 'both'; region records carry (max, sum) and no weighted sums (left unwritten); x = att (the temporal attention
    only)."""
    s, zm, z_out, _, conv, _ = P.reference(q)
    bar_t, bar_r = P.bars(q)
    R, H = P.R, P.H
    z = zbuf[:, :R]
    masked = z_out == MIN_VALUE
    assert torch.equal(z.double()[masked], z_out[masked])
    if (~masked).any():
        assert float((z.double() - z_out)[~masked].abs().max()) <= bar_r
    assert torch.isnan(zbuf[:, R:]).all()
    m, l, _ = _chunk_ref(zm, conv[:, :1].expand(-1, R, -1), P.RC)
    reg = part[:, :P.nch_r].double()
    assert float((reg[..., 0] - m).abs().max()) <= bar_r and float(((reg[..., 1] - l) / l).abs().max()) <= 2 * bar_r + 1e-6 * P.RC
    assert bool(torch.isnan(reg[..., 4:]).all())
    m, l, acc = _chunk_ref(s, conv, P.TC)
    tmp = part[:, P.nch_r:].double()
    assert float((tmp[..., 0] - m).abs().max()) <= bar_t
    att = torch.einsum("bt,bth->bh", torch.softmax(s, 1), conv)
    err = float((x.double() - att).abs().max()) / float(conv.abs().max())
    assert err <= 2 * bar_t + 1e-5, (err, bar_t)
    if xbuf.shape[1] > H:
        assert torch.isnan(xbuf[:, :H]).all() and torch.isnan(xbuf[:, 2 * H:]).all()
    return err


_ATT_CASES = [   # B, R, T, A, H, RC, TC, feat_div
    (5, 52, 10, 96, 248, 16, 16, 1),
    (5, 52, 10, 512, 248, 7, 7, 1),
    (3, 129, 480, 512, 1024, 80, 128, 1),
    (100, 1000, 10, 512, 1024, 128, 16, 1),
    (12, 52, 10, 512, 1024, 16, 16, 3),
    (128, 13, 10, 256, 248, 7, 16, 4),
]


@pytest.mark.parametrize("B,R,T,A,H,RC,TC,div", _ATT_CASES, ids=["B%d-R%d-T%d-A%d-H%d-RC%d-TC%d-div%d" % c for c in _ATT_CASES])
def test_featmap_attention_against_fp64(B, R, T, A, H, RC, TC, div):
    """gvd_op_attention_mode('featmap') without the region features: fused merge into a column window with its fp16x3 image, then the
    separate combine kernel (bit-equal), then 'both' on the same problem (its logits are the same launch arithmetic: bit-equal)."""
    P = _Attn(B, R, T, A, H, RC, TC, div, seed=B * 5 + R + T + A + H + RC + TC, mask_stride=True)
    zbuf, x, xbuf, part, ticket = _run_featmap(P, x_ld=3 * H, image=True)
    err = _check_featmap(P, zbuf, x, xbuf, part)
    print("featmap attention B=%d R=%d T=%d A=%d H=%d RC=%d TC=%d div=%d: |x err|/max|f| %.2e" % (B, R, T, A, H, RC, TC, div, err))
    assert bool((ticket == 0).all())
    zbuf2, x2, _, _, _ = _run_featmap(P, fused=False)
    assert torch.equal(zbuf2[:, :R], zbuf[:, :R]) and torch.equal(x2, x)
    zb, _, _, _, _, _, _ = P.run()
    assert torch.equal(zb, zbuf[:, :R])


@pytest.mark.parametrize("q_S", [1, 3, 4])
def test_featmap_attention_query_from_split_k_planes(q_S):
    B, R, T, A, H = 7, 52, 10, 512, 1024
    P = _Attn(B, R, T, A, H, 16, 16, seed=40 + q_S)
    g = _gen(200 + q_S)
    q_part = (torch.randn(q_S, B, 2 * A, generator=g) * 0.3).cuda()
    q_bias = (torch.randn(2 * A, generator=g) * 0.3).cuda()
    q = q_bias.expand(B, 2 * A).clone()
    for s in range(q_S):
        q += q_part[s]
    zbuf, x, xbuf, part, _ = _run_featmap(P, q_part=q_part, q_bias=q_bias, x_ld=3 * H)
    zbuf_d, x_d, _, _, _ = _run_featmap(P, q=q)
    assert torch.equal(zbuf[:, :R], zbuf_d[:, :R]) and torch.equal(x, x_d)
    _check_featmap(P, zbuf, x, xbuf, part, q=q)


def _dual_problem(P, seed):
    g = _gen(seed)
    H = P.H
    gate_w = (torch.randn(H, generator=g) * 3 / H ** 0.5).cuda()
    gate_b = (torch.randn(1, generator=g) * 0.3).cuda()
    hbuf = torch.full((P.B, H + 8), NAN)
    hbuf[:, 4:4 + H] = torch.tanh(torch.randn(P.B, H, generator=g))
    return gate_w, gate_b, hbuf.cuda()[:, 4:4 + H]


def _run_dual(P, gate, q=None, q_part=None, q_bias=None, x_ld=None, image=False):
    B, R, H = P.B, P.R, P.H
    zbuf = torch.full((B, R + 5), NAN, device="cuda")
    xbuf = torch.full((B, x_ld or H), NAN, device="cuda")
    x = xbuf[:, H:2 * H] if x_ld else xbuf
    part = torch.full((B, 2 * P.nch_r, H + 4), NAN, device="cuda")
    ticket = torch.zeros(B, dtype=torch.int32, device="cuda")
    Hp = (H + 31) // 32 * 32
    img = torch.full((B, 2 * Hp), -1, dtype=torch.int32, device="cuda") if image else None
    if q is None and q_part is None:
        q = P.q
    capi.op_attention(P.p_pool, P.pool, None, None, P.w1, P.b1, P.w2, P.b2, P.att_mask, P.out_mask, zbuf[:, :R], part, x, P.RC, P.TC,
                      q=q, q_part=q_part, q_bias=q_bias, ticket=ticket, x_pk=img[:, :Hp] if image else None, feat_div=P.div,
                      att_input_mode="dual_region", gate_w=gate[0], gate_b=gate[1], gate_h=gate[2])
    torch.cuda.synchronize()
    return zbuf, x, xbuf, part, ticket, img


def _check_dual(P, gate, zbuf, x, xbuf, part, img=None, q=None):
    """fp64: z (attention2, query slot 1, w2) and zd (attention2_dual, slot 0, w1) over the same rows and masks; records of both; the gated
    x; z_out = attention2's logits."""
    A, R, H = P.A, P.R, P.H
    d = lambda t: t.double()
    idx = torch.arange(P.B, device="cuda") // P.div
    q = d(P.q if q is None else q)
    pp, pool = d(P.p_pool)[idx], d(P.pool)[idx]
    am = P.att_mask[idx][:, 1:].bool()
    z = (torch.tanh(pp + q[:, None, A:]) @ d(P.w2) + d(P.b2)).masked_fill(am, MIN_VALUE)
    zd = (torch.tanh(pp + q[:, None, :A]) @ d(P.w1) + d(P.b1)).masked_fill(am, MIN_VALUE)
    z_out = z.masked_fill(P.out_mask[idx][:, 1:].bool(), MIN_VALUE)
    g = torch.sigmoid(d(gate[2]) @ d(gate[0]) + d(gate[1]))[:, None]
    x_ref = g * torch.einsum("br,brh->bh", torch.softmax(z, 1), pool) + (1 - g) * torch.einsum("br,brh->bh", torch.softmax(zd, 1), pool)
    bars = []
    for qq, w in ((q[:, A:], P.w2), (q[:, :A], P.w1)):
        pq = float(P.p_pool.abs().max()) + float(qq.abs().max())
        bars.append(float(w.abs().sum()) * (4e-7 + 2.0 ** -24 * (pq + A / 32 + 8)))
    zz = zbuf[:, :R]
    masked = z_out == MIN_VALUE
    assert torch.equal(zz.double()[masked], z_out[masked])
    if (~masked).any():
        assert float((zz.double() - z_out)[~masked].abs().max()) <= bars[0]
    assert torch.isnan(zbuf[:, R:]).all()
    for k, (sc, bar) in enumerate(((z, bars[0]), (zd, bars[1]))):
        m, l, acc = _chunk_ref(sc, pool, P.RC)
        got = part[:, k * P.nch_r:(k + 1) * P.nch_r].double()
        assert float((got[..., 0] - m).abs().max()) <= bar, k
        assert float(((got[..., 1] - l) / l).abs().max()) <= 2 * bar + 1e-6 * P.RC, k
        assert float(((got[..., 4:] - acc).abs() / (l[..., None] * float(pool.abs().max()))).max()) <= 2 * bar + 1e-6 * P.RC, k
    err = float((x.double() - x_ref).abs().max()) / float(pool.abs().max())
    assert err <= 2 * sum(bars) + 1e-5, (err, bars)
    if xbuf.shape[1] > H:
        assert torch.isnan(xbuf[:, :H]).all() and torch.isnan(xbuf[:, 2 * H:]).all()
    if img is not None:
        from test_gpu_tcgen05 import _decode_f16x3
        Hp = (H + 31) // 32 * 32
        val, _ = _decode_f16x3(img[:, :Hp].contiguous(), H, 4.0)
        xv = x.cpu().double().numpy()
        assert float(np.abs(val - xv).max()) <= 2.0 ** -20 * max(1.0, float(np.abs(xv).max()))
    return err, float(g.min()), float(g.max())


@pytest.mark.parametrize("B,R,T,A,H,RC,TC,div", _ATT_CASES, ids=["B%d-R%d-T%d-A%d-H%d-RC%d-TC%d-div%d" % c for c in _ATT_CASES])
def test_dual_region_attention_against_fp64(B, R, T, A, H, RC, TC, div):
    """gvd_op_attention_mode('dual_region') without frame features: both attentions from one pass, the gated merge into a column window with
    its fp16x3 image; a relaunch on the same tickets is bit-equal."""
    P = _Attn(B, R, T, A, H, RC, TC, div, seed=B * 3 + R + T + A + H + RC + TC, mask_stride=True)
    gate = _dual_problem(P, seed=B + R + A)
    zbuf, x, xbuf, part, ticket, img = _run_dual(P, gate, x_ld=3 * H, image=True)
    err, gmin, gmax = _check_dual(P, gate, zbuf, x, xbuf, part, img)
    print("dual attention B=%d R=%d A=%d H=%d RC=%d div=%d: |x err|/max|f| %.2e, g in [%.2f, %.2f]" % (B, R, A, H, RC, div, err, gmin, gmax))
    assert bool((ticket == 0).all())
    zbuf2, x2, _, _, _, _ = _run_dual(P, gate, x_ld=3 * H)
    assert torch.equal(zbuf2[:, :R], zbuf[:, :R]) and torch.equal(x2, x)
    zb, _, _, _, _, _, _ = P.run()                                    # attention2's logits are the same arithmetic as in 'both'
    assert torch.equal(zb, zbuf[:, :R])


@pytest.mark.parametrize("q_S", [1, 3, 4])
def test_dual_region_attention_query_from_split_k_planes(q_S):
    B, R, T, A, H = 7, 52, 10, 512, 1024
    P = _Attn(B, R, T, A, H, 16, 16, seed=60 + q_S)
    gate = _dual_problem(P, seed=q_S)
    g = _gen(300 + q_S)
    q_part = (torch.randn(q_S, B, 2 * A, generator=g) * 0.3).cuda()
    q_bias = (torch.randn(2 * A, generator=g) * 0.3).cuda()
    q = q_bias.expand(B, 2 * A).clone()
    for s in range(q_S):
        q += q_part[s]
    zbuf, x, xbuf, part, _, _ = _run_dual(P, gate, q_part=q_part, q_bias=q_bias)
    zbuf_d, x_d, _, _, _, _ = _run_dual(P, gate, q=q)
    assert torch.equal(zbuf[:, :R], zbuf_d[:, :R]) and torch.equal(x, x_d)
    _check_dual(P, gate, zbuf, x, xbuf, part, q=q)


def test_dual_region_attention_rejects_missing_gate():
    P = _Attn(3, 13, 4, 96, 248, 7, 7, seed=1)
    with pytest.raises(capi.GvdError):
        capi.op_attention(P.p_pool, P.pool, None, None, P.w1, P.b1, P.w2, P.b2, P.att_mask, P.out_mask, torch.empty(3, 13, device="cuda"),
                          torch.empty(3, 4, 252, device="cuda"), torch.empty(3, 248, device="cuda"), 7, 7, q=P.q,
                          ticket=torch.zeros(3, dtype=torch.int32, device="cuda"), att_input_mode="dual_region")


# ------------------------------------------------------------------------------------------------------------ decode entry points
def _greedy(model, inp):
    dev = {k: inp[k].cuda() for k in KEYS}
    B, T = inp["segs_feat"].shape[:2]
    with torch.no_grad():
        seq, logp, att2, sim = model._sample(*(dev[k] for k in KEYS), {"sample_max": 1, "beam_size": 1})
    torch.cuda.synchronize()
    return seq.cpu(), logp.cpu(), att2.cpu(), sim.cpu()


@pytest.mark.parametrize("backend", [923, 3, 0])
@pytest.mark.parametrize("name", _names("greedy"))
def test_input_mode_greedy_matches_oracle_and_reference(name, backend):
    """The three product paths of the step (923: split-K fp16x3 products, 3: tensor-core products, 0: CUDA-core products)."""
    capi.set_backend(backend)
    opt, sd, inp, model = _case(name)
    fx = load_fixture(name)
    seq, logp, att2, sim = _greedy(model, inp)
    with oracle_mode(opt) as O:
        oseq, ologp, oatt2, osim = O.sample_greedy(sd, opt, inp)
    assert torch.equal(seq, oseq) and np.array_equal(seq.numpy(), fx["seq"])
    assert _maxerr(logp, ologp) <= TOL and np.max(np.abs(logp.numpy() - fx["logp"])) <= TOL
    assert _maxerr(att2, oatt2) <= TOL and np.max(np.abs(att2.numpy() - fx["att2"])) <= TOL
    assert torch.equal(att2 == -1e8, oatt2 == -1e8)
    assert _maxerr(sim, osim) <= TOL


@pytest.mark.parametrize("name", ["featmap_greedy_small_B5", "dual_greedy_small_B5"])
def test_input_mode_host_buffer_entry_point_matches_device_path(name):
    opt, sd, inp, model = _case(name)
    seq, logp, att2, sim = _greedy(model, inp)
    pinned = {k: inp[k].pin_memory() for k in KEYS}
    out = model._native.sample_greedy_host(*(pinned[k] for k in KEYS))
    assert torch.equal(out["seq"], seq) and torch.equal(out["logp"], logp) and torch.equal(out["att2"], att2) and torch.equal(out["sim"], sim)


@pytest.mark.parametrize("name", ["featmap_greedy_small_B5", "dual_greedy_small_B5"])
def test_input_mode_decode_step_matches_oracle_step(name):
    """gvd_decode_step_fwd: one teacher-fed step at a time, h_lang and the masked logits against the oracle's step of the mode."""
    opt, sd, inp, model = _case(name)
    B, T = inp["segs_feat"].shape[:2]
    nm = model._native_model()
    dev = {k: inp[k].cuda() for k in KEYS}
    nm.prologue(*(dev[k] for k in KEYS))
    nm.reset_state(B, T)
    with oracle_mode(opt) as O:
        feats = O.prologue(sd, opt, *(inp[k] for k in ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")))
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
            assert _maxerr(h, oh) <= TOL and _maxerr(z, oz) <= TOL, t


@pytest.mark.parametrize("backend", [923, 0])
@pytest.mark.parametrize("name", ["featmap_greedy_small_B5", "featmap_greedy_T10_B3", "dual_greedy_small_B5", "dual_greedy_T10_B3"])
def test_input_mode_multinomial_matches_oracle(name, backend):
    """gvd_decode_sample against the oracle's multinomial loop with the same counter-based noise; the seed is the first whose oracle run has
    no near-tie (top-2 key gap < 1e-3) at any step."""
    capi.set_backend(backend)
    opt, sd, inp, model = _case(name)
    B, T = inp["segs_feat"].shape[:2]
    rows = np.arange(B)
    tau = 0.8
    with oracle_mode(opt) as O:
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
    assert _maxerr(logp, ologp) <= TOL and _maxerr(att2, oatt2) <= TOL


@pytest.mark.parametrize("name", _names("beam"))
def test_input_mode_beam_matches_oracle_and_reference(name):
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
def test_input_mode_mle_losses_match_reference(name):
    opt, sd, inp, model = _case(name)
    got = np.array([float(l) for l in _teacher(model, inp, "MLE")])
    assert np.max(np.abs(got - load_fixture(name)["losses"])) <= TOL


@pytest.mark.parametrize("name", _names("grd"))
def test_input_mode_grd_indices_match_reference(name):
    opt, sd, inp, model = _case(name)
    fx = load_fixture(name)
    cls_pred, att_idx, grd_idx = _teacher(model, inp, "GRD")
    assert np.array_equal(cls_pred.cpu().numpy(), fx["cls_pred"])
    assert np.array_equal(att_idx.cpu().numpy(), fx["att_idx"]) and np.array_equal(grd_idx.cpu().numpy(), fx["grd_idx"])


# ------------------------------------------------------------------------------------------------------------ training
@pytest.mark.parametrize("name", _names("train"))
def test_input_mode_training_step_against_oracle(name):
    from gvd_b200.train import TrainStep
    from gvd_b200.train_ops import NativeOps
    opt, sd, inp = build_case(CASES[name])
    with oracle_mode(opt) as O:
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
def test_input_mode_trainer_two_steps(name):
    """Trainer over NativeOps for two steps against the same Trainer over the torch mock; the tensors without a gradient (the whole region
    branch when w_att2 = w_grd = 0) come out bit-identical."""
    from gvd_b200.train import Trainer
    from gvd_b200.train_ops import NativeOps
    from ops_ref import TorchRefOps
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    a, b = Trainer(NativeOps(), sd, opt), Trainer(TorchRefOps(), sd, opt)
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
    if opt.att_input_mode == "dual_region":                            # att_embed_aux never runs: its statistics stay
        for k in ("att_embed_aux.0.running_mean", "att_embed_aux.0.running_var", "att_embed_aux.0.num_batches_tracked"):
            assert torch.equal(a.buffers[k].cpu(), sd[k]), k


def test_dual_region_module_train_mode_through_the_driver_contract():
    """model.train(); losses = model(..., 'MLE'); loss.backward(): every .grad against the oracle, no .grad on the frame branch, and the
    BatchNorm running statistics and counter untouched."""
    name = "dual_train_small_B5"
    opt, sd, inp = build_case(CASES[name])
    with oracle_mode(opt) as O:
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
    for k, p in model.named_parameters():
        if k in grads:
            assert float((p.grad.cpu() - grads[k]).abs().max()) <= 1e-4 * float(grads[k].abs().max()) + 1e-6 * scale, k
        else:
            assert p.grad is None, k
    bsd = model.state_dict()
    for k in ("att_embed_aux.0.running_mean", "att_embed_aux.0.running_var", "att_embed_aux.0.num_batches_tracked"):
        assert torch.equal(bsd[k].cpu(), sd[k]), k
