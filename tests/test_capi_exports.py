"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol
include/gvd_b200.h declares; the host mirror keeps the reference's state_dict keys; the product
path refuses to run without CUDA (no fallback)."""
import os
import re
import warnings

import pytest
import torch

import gvd_b200.synth as synth
from gvd_b200 import capi

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "grounded-video-description_b200")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "gvd_b200.h")).read()
    return sorted(set(re.findall(r"GVD_API[^;(]*?\b(gvd_\w+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = capi.lib()
    names = _declared()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), n
    assert sorted(capi.EXPORTS) == names
    assert b"sm_90a" in lib.gvd_version()


def test_state_dict_contract_matches_reference_keys():
    from gvd_b200.misc.AttModel import TopDownModel
    opt = synth.make_opt(t_attn_size=10)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    sd = synth.make_state_dict(opt)
    assert list(m.state_dict().keys()) == list(sd.keys())          # same keys, same order as the reference
    for k, v in m.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
    assert sum(v.numel() for v in sd.values()) == 68525790          # SURVEY.md 8b (+ BN counter, biases)
    m.load_state_dict(sd, strict=True)


def test_no_cpu_fallback():
    from gvd_b200.misc.AttModel import TopDownModel
    opt = synth.make_opt(t_attn_size=10, **{k: v for k, v in dict(
        vocab_size=301, detect_size=30, input_encoding_size=64, rnn_size=248, att_hid_size=96, seq_length=9,
        num_sampled_frm=4, num_prop_per_frm=13, n_vg_cls=64).items()})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt).eval()
    inp = synth.make_inputs(opt, 2)
    d = torch.zeros(2, dtype=torch.uint8)
    with pytest.raises(capi.GvdError):
        m(inp["segs_feat"], d, d, inp["num"], inp["ppls"], d, d, inp["ppls_feat"], d, inp["sample_idx"], inp["pnt_mask"],
          "sample", {"sample_max": 1, "beam_size": 1})


def test_unsupported_modes_raise():
    from gvd_b200.misc.AttModel import TopDownModel
    for bad in (dict(att_model="bogus"), dict(att_input_mode="region"), dict(t_attn_mode="bilstm"), dict(att_model="transformer", att_input_mode="x")):
        with pytest.raises(NotImplementedError):
            TopDownModel(synth.make_opt(**bad))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(synth.make_opt(att_model="transformer", att_input_mode="region"))      # the captioner picks its encoder outputs by att_input_mode
    assert any(k.startswith("cap_model.decoder.layers.1.attention.layer.wk") for k in m.state_dict())
    opt = synth.make_opt()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    with pytest.raises(ValueError):
        m(*([None] * 11), "bogus")


def test_skinny_split_plan_host_logic():
    """K-split planning of the operand-swapped decode products (pure host logic, no device call): one wave of <= 132
    (128-weight-row tile, K split) CTAs, whole 32-wide slices, >= 2 slices per split; unsupported shapes fall back (0)."""
    L = capi.lib()
    plan = L.gvd_plan_skinny_splits
    assert plan(4096, 1536, 100) == 4      # attention LSTM: [W_ih(token) | W_hh], E + H
    assert plan(4096, 3072, 100) == 4      # language LSTM: 3H
    assert plan(1024, 1024, 100) == 16     # both attention queries
    assert plan(4905, 1024, 100) == 2      # vocabulary head: 39 row tiles x 2 splits = 78 CTAs
    for nw, k, b in [(4096, 1536, 100), (4096, 3072, 100), (1024, 1024, 100), (4905, 1024, 100), (992, 320, 5)]:
        s = plan(nw, k, b)
        assert s >= 1 and k % (s * 32) == 0 and -(-nw // 128) * s <= 132 and (s == 1 or k // s >= 64)
    assert plan(4096, 1536, 129) == 0 and plan(4096, 1000, 100) == 0 and plan(64, 1024, 100) == 0


def test_h2d_chunk_plan_default_schedule():
    """Clip chunks of the host-buffer entry point (pure host logic): the sizes sum to the batch, start with ONE attention sub-batch (the first
    kernel waits for the first copy) and never shrink before the tail; a caller's array too small for the plan is an error."""
    import ctypes
    L = capi.lib()

    def plan(B, unit):
        out = (ctypes.c_int * 256)()
        n = L.gvd_plan_h2d_chunks(B, unit, out, 256)
        assert n >= 1
        return list(out[:n])
    assert plan(100, 3) == [3, 6, 9, 18, 27, 37]          # the schedule of BASELINE configs[1] (DESIGN.md 5b row 1)
    for B, unit in [(1, 1), (2, 3), (5, 3), (16, 3), (33, 3), (64, 3), (100, 1), (100, 3), (128, 3), (300, 3), (800, 3)]:
        s = plan(B, unit)
        assert sum(s) == B and all(c >= 1 for c in s)
        assert s[0] == min(B, unit) or len(s) == 1
        assert all(s[i] <= s[i + 1] for i in range(len(s) - 2))                        # non-decreasing up to the remainder chunk
        assert all(c % unit == 0 for c in s[:-1])                                       # whole sub-batches except the last chunk
    out = (ctypes.c_int * 2)()
    assert L.gvd_plan_h2d_chunks(100, 3, out, 2) == -1 and b"do not fit" in L.gvd_last_error()   # error path: status + message, no overflow


def test_training_primitive_bindings_match_the_header():
    """Every ctypes signature in gvd_b200/train_ops.py against the prototype in include/gvd_b200.h (argument count and kind):
    a mismatch here would be a crash or silent garbage on the device."""
    import ctypes
    from gvd_b200 import train_ops
    src = open(os.path.join(ROOT, "include", "gvd_b200.h")).read()
    kind = {ctypes.c_void_p: "ptr", ctypes.c_int: "int", ctypes.c_longlong: "ll", ctypes.c_float: "float"}
    protos = dict(re.findall(r"GVD_API\s+int\s+(gvd_tr_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S))
    assert set(protos) == set(train_ops._SIGS)
    for name, args in protos.items():
        want = []
        for a in [x.strip() for x in re.sub(r"/\*.*?\*/", "", args, flags=re.S).split(",")]:
            if "*" in a:
                want.append("ptr")
            elif re.match(r"(const\s+)?long long\b", a):
                want.append("ll")
            elif re.match(r"(const\s+)?float\b", a):
                want.append("float")
            elif re.match(r"(const\s+)?int\b", a):
                want.append("int")
            else:
                raise AssertionError((name, a))
        got = [kind[t] for t in train_ops._SIGS[name]]
        assert got == want, (name, got, want)


def test_training_modules_import_in_the_drop_in_layout():
    """ADVICE r1: with the package DIRECTORY on sys.path (`from misc import AttModel`, main.py:41) `__package__` is 'misc', so the training
    path must not rely on package-relative imports only.  A fresh interpreter imports everything `_forward_train` needs."""
    import subprocess
    import sys
    code = ("import sys; sys.path.insert(0, %r); import misc.model as m; import train, train_autograd, train_ops, capi; "
            "import inspect; src = inspect.getsource(m.AttModel._forward_train); assert 'from train import' in src; print('ok')" % PKG)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]
