"""The grounded beam search on the device (gvd_beam_decode_att2 / forward(..., 'sample') with eval_opt['att2_weights']): the region-attention
logits of each returned caption, gathered from the step history along the caption's ancestor chain.

  - on every beam case of the reference's fixtures: seq / logps bit for bit those of the plain beam search, logits within 1e-4 of the
    oracle's grounded beam (tests/beam_att2_ref.py);
  - at B = 100, T = 480, beam 3: per frame, the argmax of the logits is the 'GRD' teacher-forced pass's on the returned captions (near
    ties aside), and extract_grounding gives the boxes of those indices;
  - a video-indexed batch equals the per-clip call;
  - gvd_op_beam_att2_scripted against beam_att2_ref.scripted_att2: ties, a beam finishing at step 0, no beam finishing before the last
    step, L = 64."""
import gc
import warnings

import numpy as np
import pytest
import torch

import gvd_b200.synth as synth
from beam_att2_ref import BEAM_CASES, beam_case, caption_length, sample_beam_att2, scripted_att2
from beam_ref import make_script
from cases import CASES, load_fixture
from gvd_b200 import capi
from region_attn_oracle import oracle_modes
from test_gpu_attn_beam_ops import _gen

pytestmark = pytest.mark.gpu
TOL = 1e-4
KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


@pytest.fixture(autouse=True, scope="module")
def _release_models():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _maxerr(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def _model(opt, sd):
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    m.load_state_dict(sd)
    return m.cuda().eval()


def _sample(model, dev, eval_opt):
    with torch.no_grad():
        out = model._sample(*(dev[k] for k in KEYS), eval_opt)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", sorted(BEAM_CASES))
def test_grounded_beam_matches_plain_beam_and_oracle(name):
    case, opt, sd, W, inp = beam_case(name)
    K = case["beam_size"]
    fx = load_fixture(name)
    model = _model(opt, sd)
    dev = {k: inp[k].cuda() for k in KEYS}
    seq0, logp0, att0, sim0 = _sample(model, dev, {"beam_size": K})
    seq, logp, att2, sim = _sample(model, dev, {"beam_size": K, "att2_weights": True})
    assert torch.equal(seq, seq0)
    assert np.array_equal(logp.cpu().numpy().view(np.int32), logp0.cpu().numpy().view(np.int32))
    assert torch.equal(sim, sim0)
    assert np.array_equal(seq.cpu().numpy(), fx["seq"])
    B, L = seq.shape
    assert att2.shape == (B, L, model._native.R) and att2.dtype == torch.float32
    with oracle_modes(opt):
        oseq, olp, oatt, oatt2 = sample_beam_att2(W, opt, inp, K)
    assert torch.equal(seq.cpu(), oseq)
    live = oatt2 > -1e7
    scale = max(1.0, float(oatt2[live].abs().max()))            # dp / mix_mul logits are not O(1)
    assert _maxerr(att2, oatt2) <= TOL * scale
    for b, n in enumerate(caption_length(oseq)):
        assert not att2[b, n:].any()
    # the reference driver's per-frame argmax and attention softmax (main.py:364-370) run on the output as they are
    F, P = opt.num_sampled_frm, opt.num_prop_per_frm
    _, ind = torch.max(att2.view(B, L, F, P), -1)
    assert ind.shape == (B, L, F) and bool(torch.isfinite(torch.softmax(att2.view(B, L, F, P), -1)).all())
    # forward(..., 'sample') returns the logits as its second output; a greedy decode after it is undisturbed
    d = torch.zeros(B, dtype=torch.uint8, device="cuda")
    with torch.no_grad():
        seq_f, att2_f, _ = model(dev["segs_feat"], d, d, dev["num"], dev["ppls"], d, d, dev["ppls_feat"], d, dev["sample_idx"], dev["pnt_mask"],
                                 "sample", {"sample_max": 1, "beam_size": K, "att2_weights": True})
        g0 = model._sample(*(dev[k] for k in KEYS), {"sample_max": 1, "beam_size": 1})
        g1 = model._sample(*(dev[k] for k in KEYS), {"sample_max": 1, "beam_size": 1, "att2_weights": True})
    torch.cuda.synchronize()
    assert torch.equal(seq_f, seq) and torch.equal(att2_f, att2)
    for x, y in zip(g0, g1):                                    # beam_size 1: the key changes nothing
        assert torch.equal(x, y)


def test_grounded_beam_agrees_with_teacher_forced_grounding_B100_T480():
    opt = synth.make_opt(t_attn_size=480)
    sd = synth.make_state_dict(opt)
    sd["logit.bias"][0] += 3.5                                 # as beam3_T10_B4_eos: some captions end early
    model = _model(opt, sd)
    inp = synth.make_inputs(opt, 100, seed=2025, train=True)
    dev = {k: v.cuda() for k, v in inp.items()}
    B, L, F, P = 100, opt.seq_length, opt.num_sampled_frm, opt.num_prop_per_frm
    seq0, logp0, _, _ = _sample(model, dev, {"beam_size": 3})
    seq, logp, att2, _ = _sample(model, dev, {"beam_size": 3, "att2_weights": True})
    assert torch.equal(seq, seq0) and torch.equal(logp, logp0)
    n = caption_length(seq.cpu())
    assert min(n) < L                                          # some captions end early: their tails must be zero
    for b in range(B):
        assert not att2[b, n[b]:].any()
    # the 'GRD' teacher-forced pass on the returned captions (teacher_forward mode 1)
    gt_seq = seq.view(B, 1, L)
    input_seq = torch.zeros(B, 1, L + 1, 4, dtype=torch.long, device="cuda")
    with torch.no_grad():
        _, att_idx, _ = model(dev["segs_feat"], input_seq, gt_seq, dev["num"], dev["ppls"], dev["gt_boxes"], dev["mask_boxes"], dev["ppls_feat"],
                              dev["frm_mask"], dev["sample_idx"], dev["pnt_mask"], "GRD")
    torch.cuda.synchronize()
    S = att_idx.shape[1]
    assert S >= max(n)
    a = att2.view(B, L, F, P).cpu()
    mine = a.argmax(-1)
    tf = att_idx.cpu()
    rows = torch.zeros(B, L, dtype=torch.bool)
    for b in range(B):
        rows[b, :n[b]] = True
    diff = (mine[:, :S] != tf) & rows[:, :S, None]
    if bool(diff.any()):                                       # near ties only: both candidates' logits within 1e-4
        va = a[:, :S].gather(-1, mine[:, :S, :, None])[..., 0]
        vt = a[:, :S].gather(-1, tf[:, :, :, None])[..., 0]
        assert float((va - vt).abs()[diff].max()) <= TOL
    assert float(diff.float().mean()) < 0.01
    # extract_grounding on the output: the boxes of those indices
    idx, boxes = model.extract_grounding(att2, dev["ppls"])
    torch.cuda.synchronize()
    assert torch.equal(idx.cpu(), mine)
    fr = torch.arange(F)[None, None, :] * P
    want = inp["ppls"][torch.arange(B)[:, None, None], fr + mine]
    assert torch.equal(boxes.cpu(), want)


def test_grounded_beam_video_batch_equals_per_clip():
    opt = synth.make_opt(**dict(CASES["greedy_small_B5"]["opt"], t_attn_size=48))
    sd = synth.make_state_dict(opt, seed=3)
    inp = synth.make_video_inputs(opt, 100, 28, seed=11)
    model = _model(opt, sd)
    dev = {k: v.cuda() for k, v in inp.items()}
    per_clip = dict(dev, segs_feat=dev["segs_feat"][dev["video_idx"]].contiguous())
    seq, logp, att2, _ = _sample(model, dev, {"beam_size": 3, "att2_weights": True, "video_idx": dev["video_idx"]})
    seq0, logp0, att20, _ = _sample(model, per_clip, {"beam_size": 3, "att2_weights": True})
    seq_i, logp_i, _, _ = _sample(model, dev, {"beam_size": 3, "video_idx": dev["video_idx"]})
    assert torch.equal(seq, seq_i) and torch.equal(logp, logp_i)
    # as in the plain video-batch beam test: a clip whose two best continuations are closer than the tolerance may rank them either way
    same = ~(seq != seq0).any(1)
    near = (logp - logp0).abs().max(1).values <= 1e-5
    assert bool((same | near).all())
    assert _maxerr(att2[same], att20[same]) <= 1e-5 and _maxerr(logp[same], logp0[same]) <= 1e-5


SCRIPTS = [  # B, K, L, V, R, script kwargs
    (7, 3, 20, 257, 52, dict()),
    (7, 3, 20, 257, 52, dict(ties=True, no_eos=True)),
    (7, 5, 6, 40, 13, dict(eos_at=0)),
    (7, 4, 20, 257, 1000, dict(no_eos=True)),
    (100, 3, 64, 257, 1000, dict()),
    (5, 8, 64, 300, 37, dict(eos_at=40)),
    (3, 2, 1, 9, 13, dict()),
]


@pytest.mark.parametrize("B,K,L,V,R,kw", SCRIPTS)
def test_scripted_att2_matches_reference(B, K, L, V, R, kw):
    """gvd_op_beam_att2_scripted against scripted_att2 on the device's own beam_topk output (as test_scripted_beam_search): the search as
    gvd_op_beam_search_scripted returns it, and the gathered rows bit for bit (they are copies of the script's z)."""
    logits, z = make_script(B, K, L, V, R, seed=B * 100 + K * 10 + L + R, **kw)
    lt, zt = torch.from_numpy(logits).cuda(), torch.from_numpy(z).cuda()
    probe0 = torch.randn(B * K, 64, generator=_gen(B + K + L)).cuda()
    p1, p2 = probe0.clone(), probe0.clone()
    seq, lp, att, parents, att2 = capi.op_beam_att2_scripted(lt, zt, p1, K)
    seq0, lp0, att0, parents0 = capi.op_beam_search_scripted(lt, zt, p2, K)
    topv, topi = capi.op_beam_topk(lt.view(L * B * K, V), K)
    torch.cuda.synchronize()
    assert torch.equal(seq, seq0) and torch.equal(att, att0) and torch.equal(parents, parents0) and torch.equal(p1, p2)
    assert np.array_equal(lp.cpu().numpy().view(np.int32), lp0.cpu().numpy().view(np.int32))
    topk = (topv.cpu().numpy().reshape(L, B * K, K), topi.cpu().numpy().reshape(L, B * K, K))
    rseq, rlp, ratt, rpar, ratt2 = scripted_att2(logits, z, K, L, topk=topk)
    assert np.array_equal(seq.cpu().numpy(), rseq) and np.array_equal(parents.cpu().numpy(), rpar) and np.array_equal(att.cpu().numpy(), ratt)
    assert np.array_equal(att2.cpu().numpy(), ratt2)
    if kw.get("eos_at") == 0:
        assert caption_length(rseq) == [1] * B
    if kw.get("no_eos") and K < V:
        assert caption_length(rseq) == [L] * B


def test_grounded_beam_argument_checks():
    case, opt, sd, W, inp = beam_case("beam2_small_B3")
    model = _model(opt, sd)
    nm = model._native_model()
    dev = {k: inp[k].cuda() for k in KEYS}
    B, T = dev["ppls"].shape[0], dev["segs_feat"].shape[1]
    nm.prologue(*(dev[k] for k in KEYS), beam=2)            # sized for the plain beam search only
    with pytest.raises(capi.GvdError, match="att2"):
        nm.beam_decode_att2(B, T, 2, dev["pnt_mask"])
    nm.prologue(*(dev[k] for k in KEYS), beam=2, att2=True)
    with pytest.raises(capi.GvdError, match="beam_size"):
        nm.beam_decode_att2(B, T, 1, dev["pnt_mask"])
    lib = capi.lib()
    assert lib.gvd_workspace_bytes_beam_att2(nm._h, B, 0, T, 1) == 0
    base = lib.gvd_workspace_bytes_beam(nm._h, B, T, 2)
    extra = lib.gvd_workspace_bytes_beam_att2(nm._h, B, 0, T, 2) - base
    L, R = opt.seq_length, nm.R
    assert L * B * 2 * R * 4 <= extra <= L * B * 2 * (R + 1) * 4 + 3 * 256 + B * 4
