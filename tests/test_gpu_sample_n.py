"""n sampled captions per clip on the device: gvd_decode_sample_n against gvd_decode_sample on the batch repeated with repeat_interleave(n)
under the same seed, and the nn.Module surface (eval_opt['sample_n']).

The decode loop is bit-identical given the same prologue outputs.  The reference call runs the prologue on n times the clips, whose GEMMs
may then tile differently: where the prologue is row-count invariant (the small fixture configurations) every output is compared bit for
bit, elsewhere the tokens are, and the log-probabilities and attention logits to 1e-5."""
import gc
import warnings

import pytest
import torch

from cases import CASES, build_case
from input_mode_cases import INPUT_MODE_CASES
from region_attn_cases import REGION_ATTN_CASES
from vocab_cases import VOCAB_CASES
from gvd_b200 import capi, synth

pytestmark = pytest.mark.gpu

KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
TOL = 1e-5


@pytest.fixture(autouse=True, scope="module")
def _release():
    yield
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------ the decode loop
_CFG = {
    "both": CASES["greedy_small_B5"],
    "featmap": INPUT_MODE_CASES["featmap_greedy_small_B5"],
    "dual_region": INPUT_MODE_CASES["dual_greedy_small_B5"],
    "mix_mul": REGION_ATTN_CASES["mul_greedy_small_B5"],
    "dp": REGION_ATTN_CASES["dp_greedy_small_B5"],
    "dp_dual": REGION_ATTN_CASES["dp_dual_greedy_small_B5"],
    "v9001": VOCAB_CASES["v9001_greedy_small_B5"],
}
_MODELS = {}


def _model(opt, sd):
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    m.load_state_dict(sd)
    return m.cuda().eval()


def _setup(name, B=None, T=None):
    key = (name, B, T)
    if key not in _MODELS:
        _MODELS.clear()
        gc.collect()
        if name == "full":
            opt = synth.make_opt(t_attn_size=T)
            sd = synth.make_state_dict(opt, seed=1)
            inp = synth.make_inputs(opt, B, seed=77)
        else:
            case = dict(_CFG[name])
            opt, sd, inp = build_case(case)
        _MODELS[key] = (opt, inp, _model(opt, sd))
    return _MODELS[key]


def _rep(inp, n):
    return {k: v.repeat_interleave(n, 0) for k, v in inp.items()}


def _decode_n(nm, inp, n, seed, tau, video_idx=None):
    dev = {k: v.cuda() for k, v in inp.items()}
    B, T = dev["ppls"].shape[0], dev["segs_feat"].shape[1]
    nm.prologue(*(dev[k] for k in KEYS), rows=n, video_idx=video_idx)
    return [o.cpu() for o in nm.decode_sample_n(B, T, n, dev["pnt_mask"], seed, tau)]


def _decode_rep(nm, inp, n, seed, tau):
    dev = {k: v.cuda() for k, v in _rep(inp, n).items()}
    B, T = dev["ppls"].shape[0], dev["segs_feat"].shape[1]
    nm.prologue(*(dev[k] for k in KEYS))
    return [o.cpu() for o in nm.decode_sample(B, T, dev["pnt_mask"], seed, tau)]


def _assert_equal_outputs(a, b, exact=True):
    for x, y, what in zip(a, b, ("seq", "log-probs", "att2 logits")):
        assert x.shape == y.shape, what
        if exact or what == "seq":
            assert torch.equal(x, y), "%s differ (max |d| %.3g)" % (what, float((x.double() - y.double()).abs().max()))
        else:
            assert float((x.double() - y.double()).abs().max()) <= TOL, what


@pytest.mark.parametrize("tau", [0.7, 1.0, 1.5])
@pytest.mark.parametrize("name", list(_CFG))
def test_sample_n_equals_repeated_batch(name, tau):
    opt, inp, model = _setup(name)
    nm = model._native_model()
    n = 3
    _assert_equal_outputs(_decode_n(nm, inp, n, 4321, tau), _decode_rep(nm, inp, n, 4321, tau))


@pytest.mark.parametrize("T", [10, 480])
def test_sample_n_full_dims(T):
    """(B, n) = (20, 5): 100 decode rows, the split-K products off (B * n > ... rows) or on as the repeated batch has them."""
    opt, inp, model = _setup("full", 20, T)
    nm = model._native_model()
    _assert_equal_outputs(_decode_n(nm, inp, 5, 99, 1.0), _decode_rep(nm, inp, 5, 99, 1.0), exact=False)


def test_sample_n_many_rows():
    """n = 11: 55 decode rows on 5 clips."""
    opt, inp, model = _setup("both")
    nm = model._native_model()
    _assert_equal_outputs(_decode_n(nm, inp, 11, 5, 1.0), _decode_rep(nm, inp, 11, 5, 1.0), exact=False)


def test_sample_n_one_is_the_plain_call():
    opt, inp, model = _setup("both")
    nm = model._native_model()
    dev = {k: v.cuda() for k, v in inp.items()}
    B, T = dev["ppls"].shape[0], dev["segs_feat"].shape[1]
    nm.prologue(*(dev[k] for k in KEYS))
    ref = [o.cpu() for o in nm.decode_sample(B, T, dev["pnt_mask"], 8, 0.9)]
    _assert_equal_outputs(_decode_n(nm, inp, 1, 8, 0.9), ref)


def test_sample_n_video_rows():
    """video_idx: rows = events x n, equal to the per-clip batch segs_feat[video_idx] repeated n times."""
    opt = synth.make_opt(**dict(CASES["greedy_small_B5"]["opt"], t_attn_size=48))
    sd = synth.make_state_dict(opt, seed=3)
    inp = synth.make_video_inputs(opt, 12, 4, seed=11)
    model = _model(opt, sd)
    nm = model._native_model()
    vid = inp.pop("video_idx")
    got = _decode_n(nm, inp, 4, 17, 1.2, video_idx=vid.cuda())
    per_clip = dict(inp, segs_feat=inp["segs_feat"][vid].contiguous())
    _assert_equal_outputs(got, _decode_rep(nm, per_clip, 4, 17, 1.2), exact=False)


def test_replay_after_other_loops():
    """The sample_n graph is its own: greedy / plain sampling in between, and a new seed, replay it correctly."""
    opt, inp, model = _setup("both")
    nm = model._native_model()
    a = _decode_n(nm, inp, 3, 1, 1.0)
    _decode_rep(nm, inp, 3, 1, 1.0)
    b = _decode_n(nm, inp, 3, 2, 1.0)
    _assert_equal_outputs(_decode_n(nm, inp, 3, 1, 1.0), a)
    _assert_equal_outputs(b, _decode_rep(nm, inp, 3, 2, 1.0))


# ------------------------------------------------------------------------------------------------------------ the nn.Module surface
def _forward(model, inp, eval_opt):
    dev = {k: v.cuda() for k, v in inp.items()}
    d = torch.zeros(dev["ppls"].shape[0], dtype=torch.uint8, device="cuda")
    with torch.no_grad():
        return model(dev["segs_feat"], d, d, dev["num"], dev["ppls"], d, d, dev["ppls_feat"], d, dev["sample_idx"], dev["pnt_mask"], "sample",
                     eval_opt)


def test_module_shapes_and_sim_mat():
    opt, inp, model = _setup("both")
    B, L, R = inp["ppls"].shape[0], opt.seq_length, opt.num_sampled_frm * opt.num_prop_per_frm
    torch.manual_seed(5)
    seq, att2, sim = _forward(model, inp, {"sample_max": 0, "sample_n": 4, "temperature": 0.8})
    _, _, sim0 = _forward(model, inp, {"sample_max": 1})
    assert seq.shape == (B * 4, L) and att2.shape == (B * 4, L, R)
    assert sim.shape == sim0.shape and torch.equal(sim, sim0)
    torch.manual_seed(5)
    seq_b, att2_b, _ = _forward(model, inp, {"sample_max": 0, "sample_n": 4, "temperature": 0.8})
    assert torch.equal(seq, seq_b) and torch.equal(att2, att2_b)
    ind, box = model.extract_grounding(att2, inp["ppls"].cuda().repeat_interleave(4, 0))
    assert ind.shape[0] == B * 4 and box.shape[0] == B * 4


@pytest.mark.parametrize("eval_opt,exc", [
    ({"sample_max": 1, "sample_n": 2}, ValueError),
    ({"sample_max": 0, "sample_n": 2, "beam_size": 3}, ValueError),
    ({"sample_max": 0, "sample_n": 0}, ValueError),
    ({"sample_max": 0, "sample_n": 2.5}, ValueError),
    ({"sample_max": 0, "sample_n": True}, ValueError),
])
def test_module_refusals(eval_opt, exc):
    opt, inp, model = _setup("both")
    with pytest.raises(exc):
        _forward(model, inp, eval_opt)


def test_transformer_refuses_sample_n():
    opt, sd, inp = build_case(CASES["tfm_greedy_small_B5"])
    model = _model(opt, sd)
    with pytest.raises(NotImplementedError):
        _forward(model, inp, {"sample_max": 0, "sample_n": 2})
