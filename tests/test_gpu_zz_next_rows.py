"""Rows of SURVEY.md 8(f) ("next") built so far, through the C ABI.  The file name sorts last on purpose: these tests were added
late and must not mask the parity suite if one of them fails."""
import os

import numpy as np
import pytest
import torch

import gvd_oracle as O
from cases import CASES, build_case
from gvd_b200 import capi
from test_gpu_parity import _model, _sample, TOL

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,L,F,P", [(3, 5, 4, 13), (2, 20, 10, 100), (1, 1, 1, 1)])
def test_grounding_extract_against_oracle(B, L, F, P):
    """main.py:364-370: per word / frame argmax over the proposals + box gather, bit-exact (ties -> lowest index)."""
    g = torch.Generator().manual_seed(B * 100 + P)
    att2 = torch.randn(B, L, F * P, generator=g)
    if P > 1:
        att2[0, 0, :P] = -1e8                      # fully masked frame
        att2[-1, -1, 1] = att2[-1, -1, 0] = 50.0   # tie
    ppls = torch.randn(B, F * P, 7, generator=g)
    idx, boxes = capi.grounding_extract(att2.cuda(), ppls.cuda(), F, P)
    torch.cuda.synchronize()
    oidx, oboxes = O.grounding_extract(att2, ppls, F, P)
    assert torch.equal(idx.cpu(), oidx) and torch.equal(boxes.cpu(), oboxes)
    idx2, none = capi.grounding_extract(att2.cuda(), ppls.cuda(), F, P, want_boxes=False)
    assert none is None and torch.equal(idx2.cpu(), oidx)


def test_grounding_extract_on_a_decoded_batch():
    """The extraction applied to the att2 logits of a real greedy decode (small case) equals the oracle's on the oracle's logits."""
    name = "greedy_small_B5"
    opt, sd, inp = build_case(CASES[name])
    model = _model(opt, sd)
    seq, att2, sim = _sample(model, inp)
    F, P = opt.num_sampled_frm, opt.num_prop_per_frm
    idx, boxes = capi.grounding_extract(att2.contiguous(), inp["ppls"].cuda().contiguous(), F, P)
    idx_m, boxes_m = model.extract_grounding(att2, inp["ppls"].cuda())     # the nn.Module-level call a driver makes
    assert torch.equal(idx_m, idx) and torch.equal(boxes_m, boxes)
    oseq, ologp, oatt2, osim = O.sample_greedy(sd, opt, inp)
    oidx, oboxes = O.grounding_extract(att2.cpu(), inp["ppls"], F, P)          # same logits -> bit-exact
    assert torch.equal(idx.cpu(), oidx) and torch.equal(boxes.cpu(), oboxes)
    # on the oracle's own logits the choice may differ only where two logits are within the parity tolerance
    oidx2, _ = O.grounding_extract(oatt2, inp["ppls"], F, P)
    a = oatt2.reshape(*oidx2.shape, P)
    gap = (a.gather(-1, oidx2.unsqueeze(-1)) - a.gather(-1, idx.cpu().unsqueeze(-1))).squeeze(-1)
    assert float(gap.max()) <= 2 * TOL


def test_grounding_eval_against_reference_fixture_and_oracle():
    """Evaluator hit test (eval_grd_anet_entities.py:95-102): bit-exact max IoU and hits vs the reference's own outputs
    (tests/golden/grd_eval_small.npz) and vs the oracle on a larger random set."""
    fx = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "grd_eval_small.npz"))
    pred, ref, nref = (torch.from_numpy(fx[k]) for k in ("pred", "ref", "nref"))
    mx, hit = capi.grounding_eval(pred.cuda(), ref.cuda(), nref.cuda(), 0.5)
    torch.cuda.synchronize()
    assert np.array_equal(mx.cpu().numpy(), fx["max_iou"]) and np.array_equal(hit.cpu().numpy(), fx["hit"])
    g = torch.Generator().manual_seed(2)
    N, F, K = 500, 10, 9
    xy = torch.randint(0, 500, (N, F, 2), generator=g).float()
    pred = torch.cat([xy, xy + torch.randint(0, 150, (N, F, 2), generator=g).float(), torch.arange(F).float().expand(N, F).unsqueeze(-1)], -1)
    nref = torch.randint(0, K + 1, (N,), generator=g, dtype=torch.int32)
    rf = torch.randint(0, F, (N, K), generator=g)
    base = torch.gather(pred[:, :, :4], 1, rf.unsqueeze(-1).expand(N, K, 4)) + torch.randint(-30, 31, (N, K, 4), generator=g).float()
    base[:, :, 2:] = torch.maximum(base[:, :, 2:], base[:, :, :2])
    ref = torch.cat([base, rf.float().unsqueeze(-1)], -1).contiguous()
    omx, ohit = O.grounding_eval(pred, ref, nref, 0.5)
    mx, hit = capi.grounding_eval(pred.contiguous().cuda(), ref.cuda(), nref.cuda(), 0.5)
    assert torch.equal(mx.cpu(), omx) and torch.equal(hit.cpu(), ohit)
    assert 50 < int(ohit.sum()) < 450
