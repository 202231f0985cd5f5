"""ctypes binding of the C-ABI in include/gvd_b200.h (libgvd_b200.so, hand-written sm_90a CUDA).

PyTorch is used here only for device memory, streams and dtype bookkeeping: every entry point
receives raw device pointers (``tensor.data_ptr()``), sizes and the current CUDA stream.
There is no fallback: if the shared library is missing, or a tensor is not on a CUDA device,
the call raises.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgvd_b200.so")

EXPORTS = [
    "gvd_last_error", "gvd_version", "gvd_model_create", "gvd_model_create_mode", "gvd_model_create_modes", "gvd_model_create_opts", "gvd_model_destroy", "gvd_model_set_param",
    "gvd_model_num_params", "gvd_model_param_key", "gvd_model_finalize", "gvd_workspace_bytes",
    "gvd_workspace_tensor", "gvd_prologue_fwd", "gvd_decode_greedy", "gvd_decode_sample", "gvd_decode_step_fwd",
    "gvd_decode_reset_state", "gvd_sample_greedy_host", "gvd_op_linear", "gvd_op_tanh", "gvd_op_kernel_launches",
    "gvd_profile_enable", "gvd_profile_reset", "gvd_profile_count", "gvd_profile_entry",
    "gvd_op_linear_tc", "gvd_op_linear_f16ss", "gvd_op_skinny_partials", "gvd_op_reduce_lstm", "gvd_op_reduce_bias", "gvd_op_reduce_pick",
    "gvd_op_reduce_sample", "gvd_op_reduce_pick_split", "gvd_op_greedy_pick", "gvd_op_logit_pick_tc", "gvd_op_gru_layer", "gvd_op_attention", "gvd_op_attention_mode", "gvd_op_attention_form", "gvd_op_beam_topk",
    "gvd_op_row_argmax", "gvd_op_beam_search_scripted", "gvd_op_scores_tc", "gvd_op_self_attention_tc", "gvd_op_self_attention_fused", "gvd_op_lstm_step", "gvd_set_backend", "gvd_get_backend",
    "gvd_tfm_workspace_bytes", "gvd_tfm_decode_greedy", "gvd_tfm_teacher_fwd",
    "gvd_grounding_extract", "gvd_grounding_eval", "gvd_plan_skinny_splits", "gvd_plan_h2d_chunks", "gvd_workspace_bytes_beam", "gvd_beam_decode", "gvd_workspace_bytes_teacher", "gvd_teacher_fwd",
    "gvd_workspace_bytes_video", "gvd_prologue_fwd_video", "gvd_sample_greedy_host_video", "gvd_op_attention_video",
    "gvd_workspace_bytes_beam_att2", "gvd_beam_decode_att2", "gvd_op_beam_att2_scripted",
    "gvd_workspace_bytes_sample_n", "gvd_decode_sample_n", "gvd_op_attention_path",
    # training-step primitives (csrc/gvd_train.cu; bound in train_ops.py)
    "gvd_tr_adam_first_step", "gvd_tr_adam_flat", "gvd_tr_sgd_flat", "gvd_tr_adamax_flat", "gvd_tr_grad_norm", "gvd_tr_sumsq_scratch_bytes", "gvd_tr_att_scores_bwd", "gvd_tr_att_scores_fwd", "gvd_tr_att_scores_mul_bwd", "gvd_tr_att_scores_mul_fwd", "gvd_tr_bn_bwd", "gvd_tr_bn_normalize", "gvd_tr_cls_nll", "gvd_tr_colsum", "gvd_tr_count_inv", "gvd_tr_scalar_mul", "gvd_tr_dropout", "gvd_tr_ew", "gvd_tr_gather_rows", "gvd_tr_gemm_nt_batched", "gvd_tr_gru_cell_bwd", "gvd_tr_gru_cell_fwd", "gvd_tr_index_add_rows", "gvd_tr_lm_nll", "gvd_tr_ln_bwd", "gvd_tr_ln_fwd", "gvd_tr_ln_star_bwd", "gvd_tr_ln_star_fwd", "gvd_tr_lstm_cell_bwd", "gvd_tr_lstm_cell_fwd", "gvd_tr_mean_dim1", "gvd_tr_mha_bwd", "gvd_tr_mha_fwd", "gvd_tr_outer_rows", "gvd_tr_outer_rows_acc", "gvd_tr_pos_nll", "gvd_tr_rowsum", "gvd_tr_softmax_bwd", "gvd_tr_softmax_fwd", "gvd_tr_sum_all", "gvd_tr_targets", "gvd_tr_transpose",
]


class GvdError(RuntimeError):
    pass


class Dims(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in (
        "vocab_size", "detect_size", "input_encoding_size", "rnn_size", "att_hid_size", "seq_length",
        "num_sampled_frm", "num_prop_per_frm", "att_feat_size", "fc_feat_size", "obj_interact", "unk_idx")]


_lib = None


def lib():
    """Load libgvd_b200.so (once).  Fails loudly when the CUDA extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GvdError("%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(nvcc, sm_90a). gvd_b200 has no CPU or PyTorch fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp, ci, sz, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_int64
    L.gvd_last_error.restype = ctypes.c_char_p
    L.gvd_version.restype = ctypes.c_char_p
    L.gvd_model_create.argtypes = [ctypes.POINTER(Dims), ctypes.POINTER(vp)]
    L.gvd_model_create_mode.argtypes = [ctypes.POINTER(Dims), ci, ctypes.POINTER(vp)]
    L.gvd_model_create_modes.argtypes = [ctypes.POINTER(Dims), ci, ci, ctypes.POINTER(vp)]
    L.gvd_model_create_opts.argtypes = [ctypes.POINTER(Dims), ci, ci, ci, ci, ctypes.POINTER(vp)]
    L.gvd_model_destroy.argtypes = [vp]
    L.gvd_model_destroy.restype = None
    L.gvd_model_set_param.argtypes = [vp, ctypes.c_char_p, vp, sz, vp]
    L.gvd_model_num_params.argtypes = [vp]
    L.gvd_model_param_key.argtypes = [vp, ci, ctypes.POINTER(sz)]
    L.gvd_model_param_key.restype = ctypes.c_char_p
    L.gvd_model_finalize.argtypes = [vp, vp]
    L.gvd_workspace_bytes.argtypes = [vp, ci, ci]
    L.gvd_workspace_bytes.restype = sz
    L.gvd_workspace_bytes_beam.argtypes = [vp, ci, ci, ci]
    L.gvd_workspace_bytes_beam.restype = sz
    L.gvd_beam_decode.argtypes = [vp, ci, ci, ci, vp, sz, vp, vp, vp, vp, vp]
    L.gvd_workspace_bytes_beam_att2.argtypes = [vp, ci, ci, ci, ci]
    L.gvd_workspace_bytes_beam_att2.restype = sz
    L.gvd_beam_decode_att2.argtypes = [vp, ci, ci, ci, vp, sz, vp, vp, vp, vp, vp, vp]
    L.gvd_workspace_bytes_teacher.argtypes = [vp, ci, ci, ci]
    L.gvd_workspace_bytes_teacher.restype = sz
    L.gvd_teacher_fwd.argtypes = [vp, ci, ci, ci, ci, ci, vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.gvd_workspace_tensor.argtypes = [vp, vp, ci, ci, ctypes.c_char_p]
    L.gvd_workspace_tensor.restype = vp
    L.gvd_prologue_fwd.argtypes = [vp, ci, ci, vp, vp, vp, vp, vp, vp, vp, sz, vp, vp]
    L.gvd_workspace_bytes_video.argtypes = [vp, ci, ci, ci, ci, ci]
    L.gvd_workspace_bytes_video.restype = sz
    L.gvd_prologue_fwd_video.argtypes = [vp, ci, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp, vp]
    L.gvd_sample_greedy_host_video.argtypes = [vp, ci, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp]
    L.gvd_decode_greedy.argtypes = [vp, ci, ci, vp, sz, vp, vp, vp, vp, vp]
    L.gvd_decode_sample.argtypes = [vp, ci, ci, vp, sz, vp, ctypes.c_uint64, ctypes.c_float, vp, vp, vp, vp]
    L.gvd_workspace_bytes_sample_n.argtypes = [vp, ci, ci, ci, ci]
    L.gvd_workspace_bytes_sample_n.restype = sz
    L.gvd_decode_sample_n.argtypes = [vp, ci, ci, ci, vp, sz, vp, ctypes.c_uint64, ctypes.c_float, vp, vp, vp, vp]
    L.gvd_decode_step_fwd.argtypes = [vp, ci, ci, vp, sz, ci, vp, vp, vp, vp, i64, vp, vp]
    L.gvd_decode_reset_state.argtypes = [vp, ci, ci, vp, sz, vp]
    L.gvd_sample_greedy_host.argtypes = [vp, ci, ci, vp, vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp]
    L.gvd_op_linear.argtypes = [vp, i64, vp, i64, vp, vp, i64, ci, ci, ci, ci, vp]
    L.gvd_op_tanh.argtypes = [vp, vp, ci, vp]
    L.gvd_op_linear_tc.argtypes = [vp, i64, vp, i64, vp, vp, i64, ci, ci, ci, ci, vp]
    L.gvd_op_linear_f16ss.argtypes = [vp, i64, vp, i64, vp, vp, i64, vp, ci, ci, ci, ci, ci, ci, ci, vp, vp, ci, vp]
    L.gvd_op_scores_tc.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, i64, vp]
    L.gvd_op_self_attention_tc.argtypes = [vp, vp, ci, ci, ci, ci, ci, ctypes.c_float, vp, vp, ci, vp]
    L.gvd_op_self_attention_fused.argtypes = [vp, vp, ci, ci, ci, ci, ci, ctypes.c_float, vp, ctypes.c_int64, vp]
    L.gvd_grounding_extract.argtypes = [vp, vp, ci, ci, ci, ci, vp, vp, vp]
    L.gvd_plan_skinny_splits.argtypes = [ci, ci, ci]
    L.gvd_plan_h2d_chunks.argtypes = [ci, ci, vp, ci]
    L.gvd_grounding_eval.argtypes = [vp, vp, vp, ci, ci, ci, ctypes.c_float, vp, vp, vp]
    L.gvd_op_lstm_step.argtypes = [ci, ci, vp, ci, vp, i64, vp, ci, vp, i64, vp, vp, vp, vp, vp, ci, vp]
    L.gvd_op_skinny_partials.argtypes = [vp, ci, ci, vp, i64, ci, ci, ci, vp, ci, vp]
    L.gvd_op_reduce_lstm.argtypes = [vp, ci, ci, vp, ci, vp, vp, vp, vp, vp, i64, vp, i64, vp, i64, ci, ci, vp, i64, vp, i64, vp]
    L.gvd_op_reduce_bias.argtypes = [vp, ci, ci, ci, vp, vp, i64, ci, vp]
    L.gvd_op_reduce_pick.argtypes = [vp, ci, ci, vp, ci, ci, ci, vp, vp, vp, i64, vp, vp, i64, ci, vp, i64, vp, i64, vp]
    L.gvd_op_greedy_pick.argtypes = [vp, i64, ci, ci, ci, vp, vp, vp, i64, vp, vp, i64, ci, vp]
    L.gvd_op_reduce_sample.argtypes = [vp, ci, ci, vp, ci, ci, ctypes.c_float, ctypes.c_uint64, ci, vp, vp, vp, i64, vp, vp, i64, ci, vp, i64, vp]
    L.gvd_op_reduce_pick_split.argtypes = [vp, ci, ci, vp, ci, ci, ci, ci, ctypes.c_float, ctypes.c_uint64, ci, vp, vp, vp, i64, vp, vp, i64, ci, vp,
                                           i64, vp, i64, vp]
    L.gvd_op_logit_pick_tc.argtypes = [vp, i64, vp, i64, vp, ci, ci, ci, ci, vp, ci, vp, vp, vp, i64, vp, vp]
    L.gvd_op_gru_layer.argtypes = [ci, vp, vp, vp, vp, ci, ci, ci, vp, vp]
    L.gvd_op_attention.argtypes = [vp, vp, vp, vp, vp, vp, ci, vp, vp, vp, vp, vp, vp, vp, i64, vp, i64, vp, vp, vp, i64, vp, i64,
                                   ci, ci, ci, ci, ci, ci, ci, ci, vp]
    L.gvd_op_attention_mode.argtypes = L.gvd_op_attention.argtypes[:-1] + [ci, vp, vp, vp, i64, vp]
    L.gvd_op_attention_form.argtypes = L.gvd_op_attention_mode.argtypes[:-1] + [ci, vp]
    L.gvd_op_attention_video.argtypes = L.gvd_op_attention_form.argtypes[:-1] + [vp, vp, vp, vp]
    L.gvd_op_attention_path.argtypes = L.gvd_op_attention_video.argtypes[:-1] + [ci, vp]
    L.gvd_op_beam_topk.argtypes = [vp, i64, ci, ci, ci, vp, vp, vp]
    L.gvd_op_row_argmax.argtypes = [vp, i64, ci, ci, vp, vp]
    L.gvd_op_beam_search_scripted.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, ci, vp, vp, vp, vp, vp]
    L.gvd_op_beam_att2_scripted.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, ci, vp, vp, vp, vp, vp, vp]
    L.gvd_set_backend.argtypes = [ci]
    L.gvd_tfm_workspace_bytes.argtypes = [vp, ci, ci, ci, ci]
    L.gvd_tfm_workspace_bytes.restype = sz
    L.gvd_tfm_decode_greedy.argtypes = [vp, ci, ci, vp, ci, vp, ci, vp, vp, sz, vp, vp, vp]
    L.gvd_tfm_teacher_fwd.argtypes = [vp, ci, ci, vp, ci, vp, ci, vp, vp, sz, vp, vp, vp]
    L.gvd_op_kernel_launches.restype = ci
    L.gvd_profile_enable.argtypes = [ci]
    L.gvd_profile_entry.argtypes = [ci, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_longlong)]
    L.gvd_profile_entry.restype = ctypes.c_char_p
    _lib = L
    return L


def check(status):
    if status != 0:
        raise GvdError(lib().gvd_last_error().decode("utf-8", "replace"))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(t, dtype, name):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise GvdError("%s must be a CUDA tensor (gvd_b200 has no CPU path)" % name)
    if t.dtype != dtype:
        raise GvdError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise GvdError("%s must be contiguous" % name)
    return ctypes.c_void_p(t.data_ptr())


def kernel_launches():
    return int(lib().gvd_op_kernel_launches())


def profile_enable(on=True):
    lib().gvd_profile_enable(1 if on else 0)


def profile_reset():
    lib().gvd_profile_reset()


def profile_read():
    """{stage: (total_ms, launches)} — call after synchronising the stream."""
    L = lib()
    out = {}
    for i in range(L.gvd_profile_count()):
        ms, n = ctypes.c_double(), ctypes.c_longlong()
        name = L.gvd_profile_entry(i, ctypes.byref(ms), ctypes.byref(n))
        if name:
            out[name.decode()] = (ms.value, n.value)
    return out


# opt.att_input_mode of the top-down captioner -> GVD_ATT_INPUT_* (include/gvd_b200.h)
ATT_INPUT_MODES = {"both": 0, "featmap": 1, "dual_region": 2}
ATT_INPUT_REGION = 3          # GVD_ATT_INPUT_REGION: only with enable_BUTD, for the transformer captioner's encoder


def att_input_mode_code(opt):
    """The GVD_ATT_INPUT_* code of ``opt.att_input_mode`` for the top-down captioner (the transformer captioner's prologue and decode step
    do not depend on it: 'both'; with enable_BUTD the prologue builds fc7-only region features: GVD_ATT_INPUT_REGION)."""
    if getattr(opt, "att_model", "topdown") == "transformer":
        return ATT_INPUT_REGION if getattr(opt, "enable_BUTD", False) else ATT_INPUT_MODES["both"]
    return ATT_INPUT_MODES[getattr(opt, "att_input_mode", "both")]


# opt.region_attn_mode -> GVD_REGION_ATTN_* (include/gvd_b200.h): the region attention's score, AttModel.py:79-96
REGION_ATTN_MODES = {"mix": 0, "mix_mul": 1, "dp": 2}
# the reference's other values cannot run there, so they are refused with the reason
_REGION_ATTN_REFUSED = {
    "add": "'add' builds a model-level alpha_net = Linear(att_hid_size, 1) that the grounding applies to 2048-wide vectors "
           "(model.py:55-56,256-261): it fails unless att_hid_size == 2048",
    "cat": "'cat': Attention2.forward reads an undefined `xt` (AttModel.py:87)",
}


def region_attn_mode_code(opt):
    """The GVD_REGION_ATTN_* code of ``opt.region_attn_mode``.  The transformer captioner builds the same Attention2 parameters (its
    state_dict follows the mode) but its decode never runs them."""
    mode = getattr(opt, "region_attn_mode", "mix")
    if mode not in REGION_ATTN_MODES:
        raise NotImplementedError("region_attn_mode=%r: %s" % (mode, _REGION_ATTN_REFUSED.get(mode, "implemented: %s" % sorted(REGION_ATTN_MODES))))
    return REGION_ATTN_MODES[mode]


# opt.transfer_mode -> GVD_TRANSFER_* (include/gvd_b200.h): where the class side of the region-class similarity comes from (model.py:84-85,180-215)
TRANSFER_MODES = {"cls": 0, "none": 1}
# the reference's other values fail while it builds the module or runs its first forward, so they are refused with the reason
_TRANSFER_REFUSED = {
    "glove": "'glove' sizes the fc7 layer ctx2pool_grd [300, 2048] and the reference fails copying the detector's [2048, 2048] fc7 weights "
             "into it (model.py:88-89,158,177)",
    "both": "'both' makes fc7 2348 wide, so the region features are 300 columns wider than pool_embed was built for and the reference "
            "fails reshaping them to pool_feat_size (model.py:86-87,70,370)",
}


def transfer_mode_code(opt):
    """The GVD_TRANSFER_* code of ``opt.transfer_mode``."""
    mode = getattr(opt, "transfer_mode", "cls")
    if mode not in TRANSFER_MODES:
        raise NotImplementedError("transfer_mode=%r: %s" % (mode, _TRANSFER_REFUSED.get(mode, "implemented: %s" % sorted(TRANSFER_MODES))))
    return TRANSFER_MODES[mode]


def dims_from_opt(opt):
    """Size fields misc/model.py:31-58 reads from ``opt``."""
    att_model = getattr(opt, "att_model", "topdown")
    if att_model not in ("topdown", "transformer"):
        raise NotImplementedError("att_model=%r: 'topdown' and 'transformer' are on the accelerated path" % (att_model,))
    if getattr(opt, "enable_BUTD", False):
        if getattr(opt, "att_input_mode", "both") != "region":
            raise ValueError("enable_BUTD needs att_input_mode='region' (the reference asserts it, model.py:66, main.py:528-529); got %r"
                             % (getattr(opt, "att_input_mode", "both"),))
        if att_model == "topdown":
            raise NotImplementedError("enable_BUTD needs att_input_mode='region', which the top-down captioner does not run")
    if att_model == "transformer" and getattr(opt, "att_input_mode", "both") not in ("both", "featmap", "region"):
        raise NotImplementedError("att_input_mode=%r" % (opt.att_input_mode,))          # model.py:571-576
    if att_model == "topdown" and getattr(opt, "att_input_mode", "both") not in ATT_INPUT_MODES:
        raise NotImplementedError("att_input_mode=%r: the top-down captioner implements %s" % (opt.att_input_mode, sorted(ATT_INPUT_MODES)))
    region_attn_mode_code(opt)
    transfer_mode_code(opt)
    if getattr(opt, "t_attn_mode", "bigru") != "bigru":
        raise NotImplementedError("t_attn_mode=%r: only 'bigru' (the reference default, cfgs/anet_res101_vg_feat_10x100prop.yml) "
                                  "is implemented" % (opt.t_attn_mode,))
    if getattr(opt, "seq_per_img", 1) != 1:
        raise NotImplementedError("seq_per_img must be 1 (cfgs/anet_res101_vg_feat_10x100prop.yml:14)")
    return Dims(int(opt.vocab_size), int(opt.detect_size), int(opt.input_encoding_size), int(opt.rnn_size),
                int(opt.att_hid_size), int(opt.seq_length), int(opt.num_sampled_frm), int(opt.num_prop_per_frm),
                int(opt.att_feat_size), int(opt.fc_feat_size), 1 if getattr(opt, "obj_interact", False) else 0,
                int(opt.wtoi["UNK"]))


class NativeModel:
    """Owner of a ``gvd_model_t`` (packed weight arena on the current CUDA device)."""

    def __init__(self, opt):
        self._L = lib()
        self.dims = dims_from_opt(opt)
        self.att_input_mode = att_input_mode_code(opt)
        self.region_attn_mode = region_attn_mode_code(opt)
        self.transfer_mode = transfer_mode_code(opt)
        self._h = ctypes.c_void_p()
        if not torch.cuda.is_available():
            raise GvdError("gvd_b200 has no CPU path: a CUDA device is required")
        self.device = torch.cuda.current_device()      # the weight arena and every workspace live on this device
        self.butd = bool(getattr(opt, "enable_BUTD", False))
        check(self._L.gvd_model_create_opts(ctypes.byref(self.dims), self.att_input_mode, self.region_attn_mode, self.transfer_mode,
                                            int(self.butd), ctypes.byref(self._h)))
        self._live = None                              # (B, T, beam, nbox) of the prologue whose outputs sit in the workspace
        self._live_V = 0                               # ... and its video count (0: a per-clip prologue)
        self.R = self.dims.num_sampled_frm * self.dims.num_prop_per_frm
        self._ws = {}
        n = self._L.gvd_model_num_params(self._h)
        self.param_keys = []
        for i in range(n):
            numel = ctypes.c_size_t()
            key = self._L.gvd_model_param_key(self._h, i, ctypes.byref(numel)).decode()
            self.param_keys.append((key, numel.value))

    def __del__(self):
        try:
            if self._h:
                self._L.gvd_model_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass

    def _check_device(self, *tensors):
        """One process / one handle per GPU (SURVEY.md 8e): the arena was cudaMalloc'ed on `self.device`; launching on another
        current device, or with tensors of another device, would dereference foreign pointers."""
        cur = torch.cuda.current_device()
        if cur != self.device:
            raise GvdError("this gvd_b200 model lives on cuda:%d but the current device is cuda:%d — one process (and one model) per "
                           "GPU; nn.DataParallel replicas are not supported (use torch.distributed, bench.py --gpus N)" % (self.device, cur))
        for t in tensors:
            if t is not None and torch.is_tensor(t) and t.is_cuda and t.device.index != self.device:
                raise GvdError("tensor on cuda:%d passed to a model that lives on cuda:%d" % (t.device.index, self.device))

    # ---- weights
    def load_state_dict(self, sd):
        """Upload every float entry the reference state_dict holds (strict, like main.py:638)."""
        self._check_device()
        expected = dict(self.param_keys)
        keep = []
        for key, numel in self.param_keys:
            if key not in sd:
                raise GvdError("missing key in state_dict: %s" % key)
            t = sd[key].detach()
            if t.numel() != numel:
                raise GvdError("size mismatch for %s: expected %d elements, got %d" % (key, numel, t.numel()))
            t = t.to(device="cuda:%d" % self.device, dtype=torch.float32).contiguous()
            keep.append(t)
            check(self._L.gvd_model_set_param(self._h, key.encode(), ctypes.c_void_p(t.data_ptr()), numel, _stream()))
        for key in sd:
            if key not in expected and key != "att_embed_aux.0.num_batches_tracked" and not key.startswith("cap_model."):
                raise GvdError("unexpected key in state_dict: %s" % key)        # (cap_model.*: TransformerCaptioner.load_state_dict)
        check(self._L.gvd_model_finalize(self._h, _stream()))
        torch.cuda.current_stream().synchronize()
        del keep

    # ---- workspace
    def workspace(self, B, T, beam=1, nbox=0, V=None, att2=False, rows=1):
        """The (single) live workspace, sized for a decode with `beam` rows per clip and `nbox` GT boxes.  The prologue's outputs
        live INSIDE it, so a decode entry point that would need a larger allocation than the one the prologue ran in raises instead
        of silently reallocating (and then decoding from uninitialised memory): size it up front with prologue(..., beam=, nbox=).
        V: the layout of a video-indexed batch of V videos (0: per clip); None: the layout of the live prologue's batch.
        att2 (beam > 1): also the logit history of beam_decode_att2.  rows (> 1): decode_sample_n with that many sampled rows per clip."""
        self._check_device()
        key = (B, T, self.device)
        ws = self._ws.get(key)
        if V is None:
            V = self._live_V if self._live is not None and self._live[:2] == (B, T) else 0
        if V:                                      # a video-indexed prologue's layout (gvd_prologue_fwd_video)
            need = int(self._L.gvd_workspace_bytes_video(self._h, B, V, T, beam, nbox))
        else:
            need = int(self._L.gvd_workspace_bytes_beam(self._h, B, T, beam))
            if nbox:
                need = max(need, int(self._L.gvd_workspace_bytes_teacher(self._h, B, T, nbox)))
        if att2 and beam > 1:
            need = max(need, int(self._L.gvd_workspace_bytes_beam_att2(self._h, B, V, T, beam)))
        if rows > 1:
            need = max(need, int(self._L.gvd_workspace_bytes_sample_n(self._h, B, V, T, rows)))
        # the prologue lays the workspace out for one decode row per clip, and a beam layout can be the smaller one (B * beam > 128 rows
        # have no split-K slots)
        need = max(need, int(self._L.gvd_workspace_bytes_video(self._h, B, V, T, 1, 0)) if V else int(self._L.gvd_workspace_bytes(self._h, B, T)))
        if ws is not None and ws.numel() < need:
            if self._live is not None and self._live[:2] == (B, T) and (beam > 1 or nbox > 0 or rows > 1):
                raise GvdError("the workspace holding this batch's prologue outputs (sized for beam=%d, nbox=%d) is too small for the requested "
                               "decode (beam=%d, nbox=%d%s%s): call prologue(..., beam=%d, nbox=%d%s%s) first" %
                               (self._live[2], self._live[3], beam, nbox, ", att2" if att2 else "", ", rows=%d" % rows if rows > 1 else "", beam,
                                nbox, ", att2=True" if att2 else "", ", rows=%d" % rows if rows > 1 else ""))
            ws = None                              # a larger layout was requested before any prologue ran in it: reallocate
        if ws is None:
            self._live, self._live_V = None, 0
            nbytes = need
            if nbytes == 0:
                raise GvdError("bad workspace request B=%d T=%d" % (B, T))
            self._ws.clear()                      # one live workspace: sizes rarely change between calls
            ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda:%d" % self.device)
            self._ws[key] = ws
        return ws

    def workspace_tensor(self, B, T, name, shape):
        ws = self.workspace(B, T)
        p = self._L.gvd_workspace_tensor(self._h, ctypes.c_void_p(ws.data_ptr()), B, T, name.encode())
        if not p:
            raise GvdError("unknown workspace tensor %s" % name)
        off = p - ws.data_ptr()
        n = 1
        for s in shape:
            n *= s
        return ws[off:off + 4 * n].view(torch.float32).view(*shape)

    # ---- hot path
    def prologue(self, segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, want_sim=True, beam=1, nbox=0, video_idx=None, att2=False,
                 rows=1):
        """video_idx (int64 [B], CUDA): a video-indexed batch.  segs_feat then holds the frame features of V videos [V,T,F] and clip b is
        event b of video video_idx[b] with its window sample_idx[b]; every result equals the per-clip prologue on segs_feat[video_idx].
        att2: size the workspace for beam_decode_att2 as well; rows: for decode_sample_n with that many captions per clip."""
        self._check_device(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, video_idx)
        T = segs_feat.shape[1]
        B = check_video_batch(segs_feat, video_idx, ppls, num, ppls_feat, sample_idx, pnt_mask) if video_idx is not None else segs_feat.shape[0]
        V = segs_feat.shape[0] if video_idx is not None else 0
        self._live, self._live_V = None, 0
        ws = self.workspace(B, T, beam, nbox, V, att2, rows)
        sim = torch.empty(B, self.dims.detect_size + 1, self.R, dtype=torch.float32, device="cuda") if want_sim else None
        common = (_dev(ppls, torch.float32, "ppls"), _dev(num, torch.int64, "num"), _dev(ppls_feat, torch.float32, "ppls_feat"),
                  _dev(sample_idx, torch.int64, "sample_idx"))
        tail = (_dev(pnt_mask, torch.uint8, "pnt_mask"), ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                ctypes.c_void_p(sim.data_ptr()) if want_sim else None, _stream())
        if V:
            check(self._L.gvd_prologue_fwd_video(self._h, B, V, T, _dev(segs_feat, torch.float32, "segs_feat"), *common,
                                                 _dev(video_idx, torch.int64, "video_idx"), *tail))
        else:
            check(self._L.gvd_prologue_fwd(self._h, B, T, _dev(segs_feat, torch.float32, "segs_feat"), *common, *tail))
        self._live, self._live_V = (B, T, beam, nbox), V
        return sim

    def decode_greedy(self, B, T, pnt_mask):
        ws = self.workspace(B, T)
        L = self.dims.seq_length
        seq = torch.empty(B, L, dtype=torch.int64, device="cuda")
        logp = torch.empty(B, L, dtype=torch.float32, device="cuda")
        att2 = torch.empty(B, L, self.R, dtype=torch.float32, device="cuda")
        check(self._L.gvd_decode_greedy(self._h, B, T, ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                        _dev(pnt_mask, torch.uint8, "pnt_mask"), ctypes.c_void_p(seq.data_ptr()),
                                        ctypes.c_void_p(logp.data_ptr()), ctypes.c_void_p(att2.data_ptr()), _stream()))
        return seq, logp, att2

    def decode_sample(self, B, T, pnt_mask, seed, temperature=1.0):
        """Multinomial sampling (sample_max=0): the token of every step drawn from softmax(logits / temperature) with counter-based
        noise keyed by (seed, row, step); the same shapes as decode_greedy, log-probs untempered.  See gvd_decode_sample."""
        ws = self.workspace(B, T)
        L = self.dims.seq_length
        seq = torch.empty(B, L, dtype=torch.int64, device="cuda")
        logp = torch.empty(B, L, dtype=torch.float32, device="cuda")
        att2 = torch.empty(B, L, self.R, dtype=torch.float32, device="cuda")
        check(self._L.gvd_decode_sample(self._h, B, T, ctypes.c_void_p(ws.data_ptr()), ws.numel(), _dev(pnt_mask, torch.uint8, "pnt_mask"),
                                        int(seed) & 0xFFFFFFFFFFFFFFFF, float(temperature), ctypes.c_void_p(seq.data_ptr()),
                                        ctypes.c_void_p(logp.data_ptr()), ctypes.c_void_p(att2.data_ptr()), _stream()))
        return seq, logp, att2

    def decode_sample_n(self, B, T, n, pnt_mask, seed, temperature=1.0):
        """n multinomial captions per clip from one prologue (gvd_decode_sample_n): seq [B*n,L], logp [B*n,L], att2 [B*n,L,R], caption j of
        clip b in row b*n + j; equal to decode_sample on the batch repeated with repeat_interleave(n).  The prologue must have run with rows=n
        (n > 1); pnt_mask [B,R+1] per clip."""
        n = int(n)
        ws = self.workspace(B, T, rows=n)
        L = self.dims.seq_length
        seq = torch.empty(B * n, L, dtype=torch.int64, device="cuda")
        logp = torch.empty(B * n, L, dtype=torch.float32, device="cuda")
        att2 = torch.empty(B * n, L, self.R, dtype=torch.float32, device="cuda")
        check(self._L.gvd_decode_sample_n(self._h, B, T, n, ctypes.c_void_p(ws.data_ptr()), ws.numel(), _dev(pnt_mask, torch.uint8, "pnt_mask"),
                                          int(seed) & 0xFFFFFFFFFFFFFFFF, float(temperature), ctypes.c_void_p(seq.data_ptr()),
                                          ctypes.c_void_p(logp.data_ptr()), ctypes.c_void_p(att2.data_ptr()), _stream()))
        return seq, logp, att2

    def beam_decode(self, B, T, beam_size, pnt_mask):
        """All clips at once; returns (seq [B,L], logps [B,L], att2 region index [B,L])."""
        ws = self.workspace(B, T, beam_size)
        L = self.dims.seq_length
        seq = torch.empty(B, L, dtype=torch.int64, device="cuda")
        logp = torch.empty(B, L, dtype=torch.float32, device="cuda")
        att = torch.empty(B, L, dtype=torch.int64, device="cuda")
        check(self._L.gvd_beam_decode(self._h, B, T, int(beam_size), ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                      _dev(pnt_mask, torch.uint8, "pnt_mask"), ctypes.c_void_p(seq.data_ptr()),
                                      ctypes.c_void_p(logp.data_ptr()), ctypes.c_void_p(att.data_ptr()), _stream()))
        return seq, logp, att

    def beam_decode_att2(self, B, T, beam_size, pnt_mask):
        """beam_decode plus the region-attention logits of each returned caption [B,L,R] (gvd_beam_decode_att2): row t is the logit row the
        caption's own beam used to pick word t, rows after its last word are 0.  The prologue must have run with att2=True."""
        ws = self.workspace(B, T, beam_size, att2=True)
        L = self.dims.seq_length
        seq = torch.empty(B, L, dtype=torch.int64, device="cuda")
        logp = torch.empty(B, L, dtype=torch.float32, device="cuda")
        att = torch.empty(B, L, dtype=torch.int64, device="cuda")
        att2 = torch.empty(B, L, self.R, dtype=torch.float32, device="cuda")
        check(self._L.gvd_beam_decode_att2(self._h, B, T, int(beam_size), ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                           _dev(pnt_mask, torch.uint8, "pnt_mask"), ctypes.c_void_p(seq.data_ptr()),
                                           ctypes.c_void_p(logp.data_ptr()), ctypes.c_void_p(att.data_ptr()), ctypes.c_void_p(att2.data_ptr()),
                                           _stream()))
        return seq, logp, att, att2

    def teacher_forward(self, B, T, S, mode, seq, input_cls, ppls, gt_boxes, mask_boxes, frm_mask, pnt_mask):
        """'MLE' (mode 0) -> losses[4]; 'GRD' (mode 1) -> (att_idx, grd_idx, sim_target, cls_pred)."""
        nbox = gt_boxes.shape[1]
        ws = self.workspace(B, T, 1, nbox)
        NF = self.dims.num_sampled_frm
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        losses = att_idx = grd_idx = sim_target = cls_pred = None
        if mode == 0:
            losses = torch.empty(4, dtype=torch.float32, device="cuda")
        else:
            att_idx = torch.empty(B, S, NF, dtype=torch.int64, device="cuda")
            grd_idx = torch.empty(B, S, NF, dtype=torch.int64, device="cuda")
            sim_target = torch.empty(B, nbox, self.R, dtype=torch.int32, device="cuda")
            cls_pred = torch.empty(B, self.R, dtype=torch.int32, device="cuda")
        check(self._L.gvd_teacher_fwd(
            self._h, B, T, nbox, int(S), int(mode), ctypes.c_void_p(ws.data_ptr()), ws.numel(), _dev(seq, torch.int64, "seq"),
            _dev(input_cls, torch.int64, "input_cls"), _dev(ppls, torch.float32, "ppls"), _dev(gt_boxes, torch.float32, "gt_boxes"),
            _dev(mask_boxes, torch.uint8, "mask_boxes") if mask_boxes is not None else None, _dev(frm_mask, torch.uint8, "frm_mask"),
            _dev(pnt_mask, torch.uint8, "pnt_mask"), p(losses), p(att_idx), p(grd_idx), p(sim_target), p(cls_pred), _stream()))
        return losses if mode == 0 else (att_idx, grd_idx, sim_target, cls_pred)

    def reset_state(self, B, T):
        ws = self.workspace(B, T)
        check(self._L.gvd_decode_reset_state(self._h, B, T, ctypes.c_void_p(ws.data_ptr()), ws.numel(), _stream()))

    def decode_step(self, B, T, step, tokens, att_mask, out_mask, att2_out, att2_stride_b, h_lang_out=None):
        ws = self.workspace(B, T)
        check(self._L.gvd_decode_step_fwd(
            self._h, B, T, ctypes.c_void_p(ws.data_ptr()), ws.numel(), int(step), _dev(tokens, torch.int64, "tokens"),
            _dev(att_mask, torch.uint8, "att_mask"), _dev(out_mask, torch.uint8, "out_mask"),
            ctypes.c_void_p(att2_out.data_ptr()), int(att2_stride_b),
            ctypes.c_void_p(h_lang_out.data_ptr()) if h_lang_out is not None else None, _stream()))

    def sample_greedy_host(self, segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, out=None, video_idx=None):
        """End-to-end with HOST tensors (pinned recommended): H2D + prologue + loop + D2H inside.  video_idx (int64 [B], host): a
        video-indexed batch as in prologue(); segs_feat [V,T,F] then crosses PCIe once per video."""
        for n, t in (("segs_feat", segs_feat), ("ppls", ppls), ("num", num), ("ppls_feat", ppls_feat),
                     ("sample_idx", sample_idx), ("pnt_mask", pnt_mask), ("video_idx", video_idx)):
            if t is not None and (t.is_cuda or not t.is_contiguous()):
                raise GvdError("%s must be a contiguous host tensor" % n)
        T = segs_feat.shape[1]
        B = check_video_batch(segs_feat, video_idx, ppls, num, ppls_feat, sample_idx, pnt_mask) if video_idx is not None else segs_feat.shape[0]
        V = segs_feat.shape[0] if video_idx is not None else 0
        self._live, self._live_V = None, 0
        ws = self.workspace(B, T, 1, 0, V)
        L, R, NC = self.dims.seq_length, self.R, self.dims.detect_size + 1
        if out is None:
            out = dict(seq=torch.empty(B, L, dtype=torch.int64).pin_memory(),
                       logp=torch.empty(B, L, dtype=torch.float32).pin_memory(),
                       att2=torch.empty(B, L, R, dtype=torch.float32).pin_memory(),
                       sim=torch.empty(B, NC, R, dtype=torch.float32).pin_memory())
        hp = lambda t: ctypes.c_void_p(t.data_ptr())
        outs = (ctypes.c_void_p(ws.data_ptr()), ws.numel(), hp(out["seq"]), hp(out["logp"]), hp(out["att2"]),
                hp(out["sim"]) if out.get("sim") is not None else None, _stream())
        if V:
            check(self._L.gvd_sample_greedy_host_video(self._h, B, V, T, hp(segs_feat), hp(ppls), hp(num), hp(ppls_feat), hp(sample_idx),
                                                       hp(video_idx), hp(pnt_mask), *outs))
        else:
            check(self._L.gvd_sample_greedy_host(self._h, B, T, hp(segs_feat), hp(ppls), hp(num), hp(ppls_feat), hp(sample_idx), hp(pnt_mask),
                                                 *outs))
        self._live, self._live_V = (B, T, 1, 0), V
        return out


def check_video_batch(segs_feat, video_idx, ppls, num, ppls_feat, sample_idx, pnt_mask):
    """Validate a video-indexed batch: segs_feat [V,T,F] holds V videos, video_idx int64 [B] maps each of the B events to one of them, and
    the per-event tensors have B rows.  Returns B; raises ValueError."""
    if not torch.is_tensor(video_idx) or video_idx.dtype != torch.int64:
        raise ValueError("video_idx must be an int64 tensor, got %s" % (video_idx.dtype if torch.is_tensor(video_idx) else type(video_idx).__name__))
    if video_idx.dim() != 1 or video_idx.numel() < 1:
        raise ValueError("video_idx must be a non-empty 1-D tensor [B], got shape %s" % (tuple(video_idx.shape),))
    B, V = video_idx.numel(), segs_feat.shape[0]
    for n, t in (("ppls", ppls), ("num", num), ("ppls_feat", ppls_feat), ("sample_idx", sample_idx), ("pnt_mask", pnt_mask)):
        if t.shape[0] != B:
            raise ValueError("video_idx has %d events but %s has %d rows" % (B, n, t.shape[0]))
    lo, hi = int(video_idx.min()), int(video_idx.max())
    if lo < 0 or hi >= V:
        raise ValueError("video_idx values must lie in [0, %d) (segs_feat holds %d videos), got [%d, %d]" % (V, V, lo, hi))
    return B


class TfmLayer(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "self_wq", "self_wk", "self_wv", "self_wo", "self_gamma", "self_beta", "att_wq", "att_wk", "att_wv", "att_wo", "att_gamma", "att_beta",
        "ff_w1", "ff_b1", "ff_w2", "ff_b2", "ff_gamma", "ff_beta")]


class TfmWeights(ctypes.Structure):
    _fields_ = [("d_model", ctypes.c_int), ("d_hidden", ctypes.c_int), ("vocab_size", ctypes.c_int), ("n_heads", ctypes.c_int),
                ("layer", TfmLayer * 2), ("out_w", ctypes.c_void_p), ("out_b", ctypes.c_void_p)]


_TFM_KEYS = {"self_wq": "selfattn.layer.wq.weight", "self_wk": "selfattn.layer.wk.weight", "self_wv": "selfattn.layer.wv.weight",
             "self_wo": "selfattn.layer.wo.weight", "self_gamma": "selfattn.layernorm.gamma", "self_beta": "selfattn.layernorm.beta",
             "att_wq": "attention.layer.wq.weight", "att_wk": "attention.layer.wk.weight", "att_wv": "attention.layer.wv.weight",
             "att_wo": "attention.layer.wo.weight", "att_gamma": "attention.layernorm.gamma", "att_beta": "attention.layernorm.beta",
             "ff_w1": "feedforward.layer.linear1.weight", "ff_b1": "feedforward.layer.linear1.bias", "ff_w2": "feedforward.layer.linear2.weight",
             "ff_b2": "feedforward.layer.linear2.bias", "ff_gamma": "feedforward.layernorm.gamma", "ff_beta": "feedforward.layernorm.beta"}


def positional_encodings(L, H):
    """positional_encodings_like (misc/transformer.py:30-49) as the reference evaluates it under torch >= 1.5 (int64 positions / Python float ->
    fp32 true division, fp32 sin / cos): a constant [L, H] table, built once on the host by the binding."""
    pos = torch.arange(0, L)
    enc = torch.zeros(L, H)
    for c in range(H):
        if c % 2 == 0:
            enc[:, c] = torch.sin(pos / 10000 ** (c / H))
        else:
            enc[:, c] = torch.cos(pos / 10000 ** ((c - 1) / H))
    return enc


class TransformerCaptioner:
    """cap_model (misc/model.py:137-143) on the device: owns the cap_model.decoder.* weights and the decode workspace; the arithmetic is
    gvd_tfm_decode_greedy / gvd_tfm_teacher_fwd (csrc/gvd_tfm.cu)."""

    def __init__(self, d_model, vocab_size, seq_length, n_heads=6):
        self._L = lib()
        if not torch.cuda.is_available():
            raise GvdError("gvd_b200 has no CPU path: a CUDA device is required")
        self.device = torch.cuda.current_device()
        self.H, self.V, self.L, self.nh = int(d_model), int(vocab_size), int(seq_length), int(n_heads)
        self.w = None
        self._keep = []
        self._ws = None
        self.pe = positional_encodings(max(self.L, 1), self.H).to("cuda:%d" % self.device)

    def load_state_dict(self, sd, prefix="cap_model.decoder."):
        dev = "cuda:%d" % self.device
        w = TfmWeights()
        w.d_model, w.d_hidden, w.vocab_size, w.n_heads = self.H, self.H // 2, self.V, self.nh
        keep = []

        def up(key, shape):
            if key not in sd:
                raise GvdError("missing key in state_dict: %s" % key)
            t = sd[key].detach().to(device=dev, dtype=torch.float32).contiguous()
            if tuple(t.shape) != tuple(shape):
                raise GvdError("size mismatch for %s: expected %s, got %s" % (key, tuple(shape), tuple(t.shape)))
            keep.append(t)
            return t.data_ptr()
        H, DH = self.H, self.H // 2
        shapes = {"ff_w1": (DH, H), "ff_b1": (DH,), "ff_w2": (H, DH), "ff_b2": (H,)}
        for l in range(2):
            for field, key in _TFM_KEYS.items():
                shape = shapes.get(field, (H, H) if "_w" in field else (H,))
                setattr(w.layer[l], field, up("%slayers.%d.%s" % (prefix, l, key), shape))
        w.out_w = up(prefix + "out.weight", (self.V, H))
        w.out_b = up(prefix + "out.bias", (self.V,))
        self.w, self._keep = w, keep

    def _workspace(self, B, L, n0, n1):
        need = int(self._L.gvd_tfm_workspace_bytes(ctypes.byref(self.w), B, L, n0, n1))
        if need == 0:
            raise GvdError("bad transformer-captioner workspace request: %s" % (self._L.gvd_last_error() or b"").decode())
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device="cuda:%d" % self.device)
        return self._ws

    def _check(self, enc0, enc1):
        if self.w is None:
            raise GvdError("TransformerCaptioner: load_state_dict first")
        if torch.cuda.current_device() != self.device:
            raise GvdError("this captioner lives on cuda:%d but the current device is cuda:%d" % (self.device, torch.cuda.current_device()))
        for e in (enc0, enc1):
            if not (e.is_cuda and e.dtype == torch.float32 and e.is_contiguous() and e.dim() == 3 and e.shape[2] == self.H):
                raise GvdError("encoder outputs must be contiguous fp32 CUDA tensors [B, n, %d]" % self.H)
        if enc0.shape[0] != enc1.shape[0]:
            raise GvdError("encoder outputs disagree on the batch size")

    def decode_greedy(self, enc0, enc1, want_logits=False, L=None):
        """Decoder.greedy (transformer.py:214-241): prediction [B, L] int64 (+ the logits of every step [B, L, V])."""
        self._check(enc0, enc1)
        B, L = enc0.shape[0], int(L or self.L)
        if L > self.pe.shape[0]:
            self.pe = positional_encodings(L, self.H).to(self.pe.device)
        ws = self._workspace(B, L, enc0.shape[1], enc1.shape[1])
        seq = torch.empty(B, L, dtype=torch.int64, device=enc0.device)
        logits = torch.empty(B, L, self.V, dtype=torch.float32, device=enc0.device) if want_logits else None
        pe = self.pe[:L].contiguous() if self.pe.shape[0] != L else self.pe
        check(self._L.gvd_tfm_decode_greedy(ctypes.byref(self.w), B, L, ctypes.c_void_p(enc0.data_ptr()), enc0.shape[1],
                                            ctypes.c_void_p(enc1.data_ptr()), enc1.shape[1], ctypes.c_void_p(pe.data_ptr()),
                                            ctypes.c_void_p(ws.data_ptr()), ws.numel(), ctypes.c_void_p(seq.data_ptr()),
                                            ctypes.c_void_p(logits.data_ptr()) if want_logits else None, _stream()))
        return (seq, logits) if want_logits else seq

    def teacher_loss(self, enc0, enc1, seq):
        """Decoder.forward + masked cross-entropy (transformer.py:207-212,276-280), eval mode.  seq [B, S+1] int64 = [0, gt_seq]: position t is
        fed seq[:, t] and scored against seq[:, t+1] where that is != 0.  Returns the scalar loss as a (1,) tensor."""
        self._check(enc0, enc1)
        B, S = seq.shape[0], seq.shape[1] - 1
        if S > self.pe.shape[0]:
            self.pe = positional_encodings(S, self.H).to(self.pe.device)
        ws = self._workspace(B, S, enc0.shape[1], enc1.shape[1])
        loss = torch.empty(1, dtype=torch.float32, device=enc0.device)
        pe = self.pe[:S].contiguous()
        check(self._L.gvd_tfm_teacher_fwd(ctypes.byref(self.w), B, S, ctypes.c_void_p(enc0.data_ptr()), enc0.shape[1],
                                          ctypes.c_void_p(enc1.data_ptr()), enc1.shape[1], ctypes.c_void_p(pe.data_ptr()),
                                          ctypes.c_void_p(ws.data_ptr()), ws.numel(), _dev(seq, torch.int64, "seq"),
                                          ctypes.c_void_p(loss.data_ptr()), _stream()))
        return loss


def set_backend(flags):
    """0 = fp32 CUDA cores, 1 = wgmma 3xTF32 tensor cores for every GEMM-shaped stage."""
    lib().gvd_set_backend(int(flags))


def get_backend():
    return int(lib().gvd_get_backend())


def op_lstm_step(x0, w0, x1, w1, b1, b2, c_prev, backend):
    B, H = c_prev.shape
    h = torch.empty_like(c_prev)
    c = torch.empty_like(c_prev)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    check(lib().gvd_op_lstm_step(B, H, p(x0), x0.shape[1], p(w0), w0.stride(0), p(x1), x1.shape[1] if x1 is not None else 0,
                                 p(w1), w1.stride(0) if w1 is not None else 0, p(b1), p(b2), p(c_prev), p(h), p(c), backend, _stream()))
    return h, c


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _pitch(t):
    """Row pitch of a 2-D view whose rows are dense (a column window of a wider buffer); 0 for None."""
    if t is None:
        return 0
    if t.dim() != 2 or t.stride(1) != 1:
        raise GvdError("expected a 2-D tensor with dense rows")
    return t.stride(0)


def op_skinny_partials(W, X, S=0, f16_images=False, ldp=None, fill=float("nan")):
    """Split-K partial planes part [S, B, ldp] of X @ W.T (W [Nw,K] dense, X [B,K] with any row pitch), pre-filled with `fill` so
    that a caller can see which elements the product wrote.  S = 0: the planned number of splits."""
    Nw, K = W.shape
    B = X.shape[0]
    if S == 0:
        S = int(lib().gvd_plan_skinny_splits(Nw, K, B))
        if S < 1:
            raise GvdError("no split plan for %d x %d weights and %d rows" % (Nw, K, B))
    ldp = int(ldp or Nw)
    part = torch.full((S, B, ldp), fill, dtype=torch.float32, device="cuda")
    check(lib().gvd_op_skinny_partials(_dev(W, torch.float32, "W"), Nw, K, _ptr(X), _pitch(X), B, S, int(bool(f16_images)), _ptr(part), ldp,
                                       _stream()))
    return part


def op_reduce_lstm(part, c_prev, c_out, h0, h1=None, h2=None, pre=None, bias1=None, bias2=None, pk1=None, pk2=None, pre_div=1):
    """LSTMCell from partial planes part [S, B, ldp]; h0 / h1 / h2 (fp32) and pk1 / pk2 (fp16x3 words) are [B, H] column windows."""
    S, B, ldp = part.shape
    H = c_prev.shape[1]
    check(lib().gvd_op_reduce_lstm(_ptr(part), S, ldp, _ptr(pre), pre_div, _ptr(bias1), _ptr(bias2), _ptr(c_prev), _ptr(c_out), _ptr(h0), _pitch(h0),
                                   _ptr(h1), _pitch(h1), _ptr(h2), _pitch(h2), B, H, _ptr(pk1), _pitch(pk1), _ptr(pk2), _pitch(pk2), _stream()))


def op_reduce_bias(part, Nw, bias, out):
    S, B, ldp = part.shape
    check(lib().gvd_op_reduce_bias(_ptr(part), S, Nw, ldp, _ptr(bias), _ptr(out), _pitch(out), B, _stream()))


def _strided_outputs(seq, logp):
    """seq / logp: 1-D views (a column of a [B, L] buffer) sharing one element stride."""
    stride = seq.stride(0) if seq is not None else (logp.stride(0) if logp is not None else 1)
    if seq is not None and logp is not None and seq.stride(0) != logp.stride(0):
        raise GvdError("seq and logp destinations must share their stride")
    return stride


def op_reduce_pick(part, bias, V, unk, it, seq=None, logp=None, embed=None, xt=None, logits_out=None, xt_pk=None):
    S, B, ldp = part.shape
    E = embed.shape[1] if embed is not None else 0
    check(lib().gvd_op_reduce_pick(_ptr(part), S, ldp, _ptr(bias), B, V, unk, _ptr(it), _ptr(seq), _ptr(logp), _strided_outputs(seq, logp), _ptr(embed),
                                   _ptr(xt), _pitch(xt), E, _ptr(logits_out), _pitch(logits_out), _ptr(xt_pk), _pitch(xt_pk), _stream()))


def op_reduce_sample(part, bias, V, temperature, seed, step, it, seq=None, logp=None, embed=None, xt=None, xt_pk=None):
    """The multinomial sampler on partial planes part [S, B, ldp] (+ bias or None) at decode step `step`."""
    S, B, ldp = part.shape
    E = embed.shape[1] if embed is not None else 0
    check(lib().gvd_op_reduce_sample(_ptr(part), S, ldp, _ptr(bias), B, V, float(temperature), int(seed) & 0xFFFFFFFFFFFFFFFF, int(step), _ptr(it),
                                     _ptr(seq), _ptr(logp), _strided_outputs(seq, logp), _ptr(embed), _ptr(xt), _pitch(xt), E, _ptr(xt_pk),
                                     _pitch(xt_pk), _stream()))


VOCAB_GREEDY, VOCAB_SAMPLE, VOCAB_ARGMAX = 0, 1, 2


def op_reduce_pick_split(part, bias, V, mode, it, unk=-1, temperature=1.0, seed=0, step=0, seq=None, logp=None, embed=None, xt=None,
                         logits_out=None, xt_pk=None):
    """The vocabulary tail for any V on partial planes part [S, B, ldp] (+ bias or None): mode VOCAB_GREEDY (top-2 + UNK rule),
    VOCAB_SAMPLE (the multinomial draw at (temperature, seed, step)) or VOCAB_ARGMAX (first maximum)."""
    S, B, ldp = part.shape
    E = embed.shape[1] if embed is not None else 0
    check(lib().gvd_op_reduce_pick_split(_ptr(part), S, ldp, _ptr(bias), B, V, int(mode), int(unk), float(temperature),
                                         int(seed) & 0xFFFFFFFFFFFFFFFF, int(step), _ptr(it), _ptr(seq), _ptr(logp), _strided_outputs(seq, logp),
                                         _ptr(embed), _ptr(xt), _pitch(xt), E, _ptr(logits_out), _pitch(logits_out), _ptr(xt_pk), _pitch(xt_pk),
                                         _stream()))


def op_greedy_pick(logits, unk, it, seq=None, logp=None, embed=None, xt=None):
    B, V = logits.shape
    E = embed.shape[1] if embed is not None else 0
    check(lib().gvd_op_greedy_pick(_ptr(logits), _pitch(logits), B, V, unk, _ptr(it), _ptr(seq), _ptr(logp), _strided_outputs(seq, logp), _ptr(embed),
                                   _ptr(xt), _pitch(xt), E, _stream()))


def op_logit_pick_tc(h, W, bias, unk, it, seq=None, logp=None, embed=None, xt=None):
    """Vocabulary head h [B,K] @ W [V,K].T + bias with the sampler fused into the GEMM epilogue; xt [B,E] dense."""
    B, K = h.shape
    V = W.shape[0]
    E = embed.shape[1] if embed is not None else 0
    if xt is not None and _pitch(xt) != E:
        raise GvdError("logit_pick_tc writes xt with pitch E")
    check(lib().gvd_op_logit_pick_tc(_ptr(h), _pitch(h), _ptr(W), _pitch(W), _ptr(bias), B, V, K, unk, _ptr(embed), E, _ptr(it), _ptr(seq), _ptr(logp),
                                     _strided_outputs(seq, logp), _ptr(xt), _stream()))


def op_gru_layer(path, gi, Whh, bhh, sample_idx=None):
    """One bidirectional GRU layer from gi [B,T,6G]; returns out [B,T,2G] (pre-filled with NaN: the layer writes every element)."""
    B, T, G6 = gi.shape
    G = G6 // 6
    out = torch.full((B, T, 2 * G), float("nan"), dtype=torch.float32, device="cuda")
    check(lib().gvd_op_gru_layer(int(path), _dev(gi, torch.float32, "gi"), _dev(Whh, torch.float32, "Whh"), _dev(bhh, torch.float32, "bhh"),
                                 _dev(sample_idx, torch.int64, "sample_idx") if sample_idx is not None else None, B, T, G, _ptr(out), _stream()))
    return out


def op_attention(p_pool, pool, p_conv, conv, w1, b1, w2, b2, att_mask, out_mask, z_out, partial, x_out, RC, TC, q=None, q_part=None,
                 q_bias=None, ticket=None, x_pk=None, feat_div=1, att_input_mode=None, gate_w=None, gate_b=None, gate_h=None,
                 region_attn_mode=None, _video=None, path=None):
    """The decode attention of B query rows through gvd_op_attention.  Features [B / feat_div, N, A | H]; q [B, 2A] or its split-K planes
    q_part [q_S, B, 2A] + q_bias [2A]; att_mask [B / feat_div, R+1]; out_mask [B / feat_div, R+1] or a [B / feat_div, R+1] column window
    of a wider mask (its row pitch is passed); z_out [B, R] and x_out [B, H] (x_pk [B, rup32(H)] int32 words) may be column windows of
    wider buffers; partial [B, nch, H+4]; ticket [B] int32 (None: the separate combine kernel).  att_input_mode 'both' / 'featmap'
    (None: gvd_op_attention, i.e. 'both'); with 'featmap' x_out = att and `pool` may be None.  'dual_region': q = [attention2_dual query |
    attention2 query], w1 / b1 the dual alpha_net, p_conv / conv may be None, partial [B, 2 nch_r, H+4], the gate gate_w [H], gate_b [1] over
    the rows of gate_h [B, H] (dense rows, any pitch).  region_attn_mode 'mix' / 'mix_mul' / 'dp' (None: 'mix' through gvd_op_attention(_mode));
    in 'dp' the region alpha_net (w2 / b2, and w1 / b1 in 'dual_region') may be None.  path 0 / 1: the per-row or the row-grouped kernel
    through gvd_op_attention_path (None: the entry the other arguments select, which runs the per-row kernel)."""
    Bf, R, A = p_pool.shape
    T, H = (conv.shape[1], conv.shape[2]) if conv is not None else (1, x_out.shape[-1])
    B = (q if q is not None else q_part[0]).shape[0]
    q_S = q_part.shape[0] if q_part is not None else 0
    if out_mask.stride(1) != 1 or att_mask.stride(1) != 1 or att_mask.stride(0) != R + 1:
        raise GvdError("masks must have dense rows, att_mask a pitch of R+1")
    args = (_dev(p_pool, torch.float32, "p_pool"), _dev(pool, torch.float32, "pool") if pool is not None else None,
            _dev(p_conv, torch.float32, "p_conv") if p_conv is not None else None, _dev(conv, torch.float32, "conv") if conv is not None else None, _ptr(q), _ptr(q_part), q_S, _ptr(q_bias), _ptr(w1), _ptr(b1),
            _ptr(w2), _ptr(b2), _ptr(att_mask), _ptr(out_mask), out_mask.stride(0), _ptr(z_out), _pitch(z_out), _ptr(partial), _ptr(ticket),
            _ptr(x_out), _pitch(x_out), _ptr(x_pk), _pitch(x_pk), B, R, T, A, H, int(RC), int(TC), int(feat_div))
    if path is not None:
        vid, win, cb = _video if _video is not None else (None, None, None)
        check(lib().gvd_op_attention_path(*args, ATT_INPUT_MODES[att_input_mode or "both"], _ptr(gate_w), _ptr(gate_b), _ptr(gate_h),
                                          _pitch(gate_h), REGION_ATTN_MODES[region_attn_mode or "mix"],
                                          _dev(vid, torch.int64, "video_idx") if vid is not None else None,
                                          _dev(win, torch.int64, "sample_idx") if win is not None else None,
                                          _dev(cb, torch.float32, "ctx_bias") if cb is not None else None, int(path), _stream()))
    elif _video is not None:
        vid, win, cb = _video
        check(lib().gvd_op_attention_video(*args, ATT_INPUT_MODES[att_input_mode or "both"], _ptr(gate_w), _ptr(gate_b), _ptr(gate_h),
                                           _pitch(gate_h), REGION_ATTN_MODES[region_attn_mode or "mix"], _dev(vid, torch.int64, "video_idx"),
                                           _dev(win, torch.int64, "sample_idx"), _dev(cb, torch.float32, "ctx_bias"), _stream()))
    elif region_attn_mode is not None:
        check(lib().gvd_op_attention_form(*args, ATT_INPUT_MODES[att_input_mode or "both"], _ptr(gate_w), _ptr(gate_b), _ptr(gate_h),
                                          _pitch(gate_h), REGION_ATTN_MODES[region_attn_mode], _stream()))
    elif att_input_mode is None:
        check(lib().gvd_op_attention(*args, _stream()))
    else:
        check(lib().gvd_op_attention_mode(*args, ATT_INPUT_MODES[att_input_mode], _ptr(gate_w), _ptr(gate_b), _ptr(gate_h), _pitch(gate_h),
                                          _stream()))


def op_attention_video(video_idx, sample_idx, ctx_bias, *args, **kw):
    """op_attention over video-level frame features (gvd_op_attention_video): p_conv / conv [V, T, A | H] unmasked, video_idx [B / feat_div]
    int64, sample_idx [B / feat_div, 2] the windows, ctx_bias [A].  Equals op_attention on p_conv / conv gathered by video_idx with the rows
    outside each window set to (ctx_bias, 0)."""
    kw = dict(kw, _video=(video_idx, sample_idx, ctx_bias))
    op_attention(*args, **kw)


def op_beam_topk(logits, K):
    """(topv [rows, K] float32, topi [rows, K] int32) of logits [rows, V] (dense rows, any pitch), outputs pre-filled with NaN / -1."""
    rows, V = logits.shape
    topv = torch.full((rows, K), float("nan"), dtype=torch.float32, device="cuda")
    topi = torch.full((rows, K), -1, dtype=torch.int32, device="cuda")
    check(lib().gvd_op_beam_topk(_ptr(logits), _pitch(logits), rows, V, int(K), _ptr(topv), _ptr(topi), _stream()))
    return topv, topi


def op_row_argmax(z):
    """idx [rows] int32 (pre-filled with -1) = first index of each row maximum of z [rows, R]."""
    rows, R = z.shape
    idx = torch.full((rows,), -1, dtype=torch.int32, device="cuda")
    check(lib().gvd_op_row_argmax(_ptr(z), _pitch(z), rows, R, _ptr(idx), _stream()))
    return idx


def op_beam_search_scripted(logits, z, probe, K):
    """The beam bookkeeping of gvd_beam_decode on scripted logits [L, B*K, V] and region scores [L+1, B*K, R]; probe [B*K, H] is reordered
    in place.  Returns seq [B, L] int64, logp [B, L], att2_idx [B, L] int64 and parents [L, B*K] int32, pre-filled with sentinels."""
    L, BK, V = logits.shape
    R, H = z.shape[2], probe.shape[1]
    B = BK // K
    seq = torch.full((B, L), -7, dtype=torch.int64, device="cuda")
    logp = torch.full((B, L), float("nan"), dtype=torch.float32, device="cuda")
    att = torch.full((B, L), -7, dtype=torch.int64, device="cuda")
    parents = torch.full((L, BK), -7, dtype=torch.int32, device="cuda")
    check(lib().gvd_op_beam_search_scripted(_dev(logits, torch.float32, "logits"), _dev(z, torch.float32, "z"), _dev(probe, torch.float32, "probe"),
                                            B, int(K), L, V, R, H, _ptr(seq), _ptr(logp), _ptr(att), _ptr(parents), _stream()))
    return seq, logp, att, parents


def op_beam_att2_scripted(logits, z, probe, K):
    """op_beam_search_scripted plus att2 [B, L, R] (pre-filled with NaN): the rows of z the returned caption used (gvd_op_beam_att2_scripted)."""
    L, BK, V = logits.shape
    R, H = z.shape[2], probe.shape[1]
    B = BK // K
    seq = torch.full((B, L), -7, dtype=torch.int64, device="cuda")
    logp = torch.full((B, L), float("nan"), dtype=torch.float32, device="cuda")
    att = torch.full((B, L), -7, dtype=torch.int64, device="cuda")
    parents = torch.full((L, BK), -7, dtype=torch.int32, device="cuda")
    att2 = torch.full((B, L, R), float("nan"), dtype=torch.float32, device="cuda")
    check(lib().gvd_op_beam_att2_scripted(_dev(logits, torch.float32, "logits"), _dev(z, torch.float32, "z"), _dev(probe, torch.float32, "probe"),
                                          B, int(K), L, V, R, H, _ptr(seq), _ptr(logp), _ptr(att), _ptr(parents), _ptr(att2), _stream()))
    return seq, logp, att, parents, att2


def op_linear(A, W, bias=None, act=0, tc=False):
    """C = act(A @ W.T + bias) through gvd_op_linear / gvd_op_linear_tc (parity tests)."""
    M, K = A.shape
    N = W.shape[0]
    C = torch.empty(M, N, dtype=torch.float32, device="cuda")
    fn = lib().gvd_op_linear_tc if tc else lib().gvd_op_linear
    check(fn(_dev(A, torch.float32, "A"), A.stride(0), _dev(W, torch.float32, "W"), W.stride(0),
                              _dev(bias, torch.float32, "bias") if bias is not None else None,
                              ctypes.c_void_p(C.data_ptr()), C.stride(0), M, N, K, act, _stream()))
    return C


def op_linear_f16ss(A, W, bias=None, act=0, want_img=False, want_c=True, qkv=None):
    """The conversion-free persistent GEMM on its own; returns C [M,N] and / or the fp16x3 image of C as int32 words [M, rup32(N)].
    qkv = (nh, hs, R, C, k_img, vt_img, ref): the region encoder's Q|K|V projection into the caller's buffers (C [M, N] fp32, k_img
    [M, nh, rup32(hs)] and vt_img [M / R, nh * hs, rup32(R)] int32 words); ref=True builds the images from the fp32 product with the
    separate pack passes (and writes all of C), else the projection's epilogue writes them (and only Q, C[:, :nh * hs]).  Returns None."""
    M, K = A.shape
    N = W.shape[0]
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    if qkv is not None:
        nh, hs, R, C, k_img, vt_img, ref = qkv
        check(lib().gvd_op_linear_f16ss(p(A), A.stride(0), p(W), W.stride(0), None, p(C), C.stride(0), None, M, N, K, 0,
                                        nh, hs, R, p(k_img), p(vt_img), int(bool(ref)), _stream()))
        return None
    C = torch.empty(M, N, dtype=torch.float32, device="cuda") if want_c else None
    img = torch.empty(M, (N + 31) // 32 * 32, dtype=torch.int32, device="cuda") if want_img else None
    check(lib().gvd_op_linear_f16ss(p(A), A.stride(0), p(W), W.stride(0), p(bias), p(C), N, p(img), M, N, K, int(act),
                                    0, 0, 0, None, None, 0, _stream()))
    return (C, img) if want_img else C


def op_scores_tc(A, W, nh, hs):
    """C[b,h] = A[b][:, h*hs:(h+1)*hs] @ W[b][:, h*hs:(h+1)*hs].T through the tensor-core score product."""
    nb, M, ld = A.shape
    N = W.shape[1]
    C = torch.empty(nb, nh, M, N, dtype=torch.float32, device="cuda")
    check(lib().gvd_op_scores_tc(_dev(A, torch.float32, "A"), _dev(W, torch.float32, "W"), ctypes.c_void_p(C.data_ptr()),
                                 nb, nh, M, N, hs, ld, _stream()))
    return C


def op_self_attention_tc(qkv, nh, hs, scale, debug=False, E=None, F=None, stages=3):
    """concat_h softmax(Q_h K_h^T * scale) V_h for qkv [nb, R, 3*HP] through the fused wgmma attention pair.
    debug=True also returns the softmax as stored: numerators E [nb,nh,R,R] and group factors F [nb,nh,ceil(R/32),R];
    stages=1 runs only the score kernel, stages=2 only P.V on caller-provided E / F."""
    nb, R, three_hp = qkv.shape
    HP = three_hp // 3
    out = torch.zeros(nb, R, HP, dtype=torch.float32, device="cuda")
    if E is None:
        E = torch.zeros(nb, nh, R, R, dtype=torch.float32, device="cuda")
    if F is None:
        F = torch.zeros(nb, nh, (R + 31) // 32, R, dtype=torch.float32, device="cuda")
    check(lib().gvd_op_self_attention_tc(_dev(qkv, torch.float32, "qkv"), ctypes.c_void_p(out.data_ptr()), nb, nh, R, hs, HP,
                                         float(scale), _dev(E, torch.float32, "E"), _dev(F, torch.float32, "F"), int(stages), _stream()))
    return (out, E, F) if debug else out


def op_self_attention_fused(qkv, nh, hs, scale, img=None):
    """concat_h softmax(Q_h K_h^T * scale) V_h for qkv [nb, R, 3*HP] through the fused self-attention kernel.  Returns out [nb, R, HP]
    (fp32); with img (an int32 tensor [nb*R, img_ld]) the kernel stores the fp16x3 operand image of the output there instead and out is
    left as allocated (zeros)."""
    nb, R, three_hp = qkv.shape
    HP = three_hp // 3
    out = torch.zeros(nb, R, HP, dtype=torch.float32, device="cuda")
    img_ptr, img_ld = None, 0
    if img is not None:
        if img.dtype != torch.int32 or not img.is_cuda or not img.is_contiguous() or img.dim() != 2 or img.shape[0] != nb * R:
            raise ValueError("img must be a contiguous CUDA int32 tensor [nb*R, img_ld]")
        img_ptr, img_ld = ctypes.c_void_p(img.data_ptr()), img.shape[1]
    check(lib().gvd_op_self_attention_fused(_dev(qkv, torch.float32, "qkv"), ctypes.c_void_p(out.data_ptr()), nb, nh, R, hs, HP,
                                            float(scale), img_ptr, int(img_ld), _stream()))
    return out


def grounding_extract(att2, ppls, num_frames, num_prop, want_boxes=True):
    """main.py:364-370 on the device: att2 [B,L,F*P] logits, ppls [B,F*P,7] -> (idx [B,L,F] int64, boxes [B,L,F,7] or None)."""
    B, Lw, R = att2.shape
    if R != num_frames * num_prop or tuple(ppls.shape) != (B, R, 7):
        raise GvdError("grounding_extract: att2 [B,L,F*P] and ppls [B,F*P,7] expected, got %s and %s" % (tuple(att2.shape), tuple(ppls.shape)))
    idx = torch.empty(B, Lw, num_frames, dtype=torch.int64, device="cuda")
    boxes = torch.empty(B, Lw, num_frames, 7, dtype=torch.float32, device="cuda") if want_boxes else None
    check(lib().gvd_grounding_extract(_dev(att2, torch.float32, "att2"), _dev(ppls, torch.float32, "ppls"), B, Lw, num_frames, num_prop,
                                      ctypes.c_void_p(idx.data_ptr()), ctypes.c_void_p(boxes.data_ptr()) if want_boxes else None, _stream()))
    return idx, boxes


def grounding_eval(pred, ref, nref, iou_thresh=0.5):
    """Evaluator hit test on the device: pred [N,F,5], ref [N,K,5], nref [N] int32 -> (max_iou [N] float32, hit [N] uint8)."""
    N, F, _ = pred.shape
    K = ref.shape[1]
    mx = torch.empty(N, dtype=torch.float32, device="cuda")
    hit = torch.empty(N, dtype=torch.uint8, device="cuda")
    check(lib().gvd_grounding_eval(_dev(pred, torch.float32, "pred"), _dev(ref, torch.float32, "ref"), _dev(nref, torch.int32, "nref"),
                                   N, F, K, float(iou_thresh), ctypes.c_void_p(mx.data_ptr()), ctypes.c_void_p(hit.data_ptr()), _stream()))
    return mx, hit


def op_tanh(x):
    y = torch.empty_like(x)
    check(lib().gvd_op_tanh(_dev(x, torch.float32, "x"), ctypes.c_void_p(y.data_ptr()), x.numel(), _stream()))
    return y
