"""Deterministic synthetic `opt`, weights and clip tensors for the caption-decode hot path.

Replaces (for tests / bench / smoke) the 216 GB dataset the reference's
``misc/dataloader_anet.py:175-354`` reads; the tensor contract (names, dtypes, shapes, mask
conventions) is the one ``main.py:213-232,344-350`` hands to ``model.forward``.

Everything is generated with ``numpy.random.RandomState`` keyed by (seed, name) so the same
tensors can be rebuilt bit-identically on any box — the golden fixtures under ``tests/golden``
store only reference OUTPUTS, never weights or inputs.
"""
import types
import zlib

import numpy as np
import torch

DEFAULTS = dict(
    vocab_size=4905, detect_size=431, input_encoding_size=512, rnn_size=1024, num_layers=2,
    drop_prob_lm=0.5, seq_length=20, fc_feat_size=3072, att_feat_size=2048, att_hid_size=512,
    seq_per_img=1, att_input_mode="both", transfer_mode="cls", test_mode=False, enable_BUTD=False,
    w_att2=0.1, w_grd=0.0, w_cls=0.1, num_sampled_frm=10, num_prop_per_frm=100, att_model="topdown",
    region_attn_mode="mix", t_attn_size=480, obj_interact=True, t_attn_mode="bigru",
    enable_visdom=False, visdom_server="", id="synthetic", n_vg_cls=1601, grad_clip=0.1,
)


def _rs(seed, name):
    return np.random.RandomState((zlib.crc32(name.encode()) ^ (seed * 2654435761)) & 0x7FFFFFFF)


def make_opt(seed=0, **overrides):
    """Bare namespace with the fields ``misc/model.py:31-58`` reads (SURVEY.md 8b)."""
    cfg = dict(DEFAULTS)
    cfg.update(overrides)
    opt = types.SimpleNamespace(**cfg)
    D, V = opt.detect_size, opt.vocab_size
    opt.itod = {i: "det%d" % i for i in range(1, D + 1)}
    opt.wtoi = {"UNK": str(V - 1)}
    opt.vg_cls = ["vg%d" % i for i in range(opt.n_vg_cls)]
    opt.glove_clss = torch.from_numpy(_rs(seed, "glove_clss").standard_normal((D + 1, 300)).astype(np.float32))
    opt.glove_vg_cls = torch.from_numpy(
        _rs(seed, "glove_vg_cls").standard_normal((opt.n_vg_cls, 300)).astype(np.float32))
    return opt


def make_detectron(opt, seed=0):
    """Stand-ins for data/detectron_weights/*.pkl (misc/model.py:173-185)."""
    f = opt.att_feat_size
    return dict(
        fc7_w=(_rs(seed, "fc7_w").standard_normal((f, f)) * 0.02).astype(np.float32),
        fc7_b=(_rs(seed, "fc7_b").standard_normal((f,)) * 0.02).astype(np.float32),
        cls_score_w=(_rs(seed, "cls_score_w").standard_normal((opt.n_vg_cls, 2048)) * 0.02).astype(np.float32),
        cls_score_b=(_rs(seed, "cls_score_b").standard_normal((opt.n_vg_cls,)) * 0.02).astype(np.float32),
    )


def state_dict_spec(opt):
    """(key, shape, init-kind, fan) for every entry of the reference state_dict, in its order."""
    H, A, E, V, D = opt.rnn_size, opt.att_hid_size, opt.input_encoding_size, opt.vocab_size, opt.detect_size
    F = opt.att_feat_size
    fc = opt.fc_feat_size + 50
    pool = F if getattr(opt, "enable_BUTD", False) else F + 300 + D + 1      # BUTD: pool_embed reads fc7 alone (model.py:65-69)
    G = H // 2
    spec = []

    def lin(name, out, inp, bias=True):
        spec.append((name + ".weight", (out, inp), "uniform", inp))
        if bias:
            spec.append((name + ".bias", (out,), "uniform", inp))

    if getattr(opt, "transfer_mode", "cls") == "cls":                  # 'none' has no class bias (model.py:180-215)
        spec.append(("vis_classifiers_bias", (D + 1,), "normal", 50.0))
    lin("loc_fc.0", 300, 5)
    spec.append(("embed.0.weight", (V, E), "normal", 1.0))
    spec.append(("vis_embed.0.weight", (D + 1, 2048), "normal", 50.0))
    lin("fc_embed.0", H, fc)
    lin("seg_info_embed.0", 50, 4)
    lin("att_embed.0.0", H // 2, 2048)
    lin("att_embed.1.0", H // 2, 1024)
    spec.append(("att_embed_aux.0.weight", (H,), "gamma", 0))
    spec.append(("att_embed_aux.0.bias", (H,), "normal", 10.0))
    spec.append(("att_embed_aux.0.running_mean", (H,), "normal", 10.0))
    spec.append(("att_embed_aux.0.running_var", (H,), "var", 0))
    spec.append(("att_embed_aux.0.num_batches_tracked", (), "count", 0))
    lin("pool_embed.0", H, pool)
    lin("ctx2att", A, H)
    lin("ctx2pool", A, H)
    lin("logit", V, H)
    if opt.obj_interact:
        for l in range(2):
            p = "obj_interact.encoder.layers.%d." % l
            for w in ("wq", "wk", "wv", "wo"):
                lin(p + "selfattn.layer." + w, H, H, bias=False)
            spec.append((p + "selfattn.layernorm.gamma", (H,), "gamma", 0))
            spec.append((p + "selfattn.layernorm.beta", (H,), "normal", 10.0))
            lin(p + "feedforward.layer.linear1", H // 2, H)
            lin(p + "feedforward.layer.linear2", H, H // 2)
            spec.append((p + "feedforward.layernorm.gamma", (H,), "gamma", 0))
            spec.append((p + "feedforward.layernorm.beta", (H,), "normal", 10.0))
    if getattr(opt, "att_model", "topdown") == "transformer":           # cap_model = TransformerDecoder (model.py:137-143), between obj_interact and context_enc in the state_dict
        for l in range(2):
            p = "cap_model.decoder.layers.%d." % l
            for blk in ("selfattn", "attention"):
                for w in ("wq", "wk", "wv", "wo"):
                    lin(p + blk + ".layer." + w, H, H, bias=False)
                spec.append((p + blk + ".layernorm.gamma", (H,), "gamma", 0))
                spec.append((p + blk + ".layernorm.beta", (H,), "normal", 10.0))
            lin(p + "feedforward.layer.linear1", H // 2, H)
            lin(p + "feedforward.layer.linear2", H, H // 2)
            spec.append((p + "feedforward.layernorm.gamma", (H,), "gamma", 0))
            spec.append((p + "feedforward.layernorm.beta", (H,), "normal", 10.0))
        lin("cap_model.decoder.out", V, H)
    for l in range(2):
        for sfx in ("", "_reverse"):
            inp = H if l == 0 else 2 * G
            spec.append(("context_enc.weight_ih_l%d%s" % (l, sfx), (3 * G, inp), "uniform", G))
            spec.append(("context_enc.weight_hh_l%d%s" % (l, sfx), (3 * G, G), "uniform", G))
            spec.append(("context_enc.bias_ih_l%d%s" % (l, sfx), (3 * G,), "uniform", G))
            spec.append(("context_enc.bias_hh_l%d%s" % (l, sfx), (3 * G,), "uniform", G))
    lin("ctx2pool_grd.0", 2048, F)
    for name, inp in (("att_lstm", E + H), ("lang_lstm", 2 * H)):
        spec.append(("core.%s.weight_ih" % name, (4 * H, inp), "uniform", H))
        spec.append(("core.%s.weight_hh" % name, (4 * H, H), "uniform", H))
        spec.append(("core.%s.bias_ih" % name, (4 * H,), "uniform", H))
        spec.append(("core.%s.bias_hh" % name, (4 * H,), "uniform", H))
    region_alpha = getattr(opt, "region_attn_mode", "mix") != "dp"      # 'dp': Attention2 has no alpha_net (AttModel.py:62-65)
    for name in ("attention", "attention2"):
        lin("core.%s.h2att" % name, A, H)
        if name == "attention" or region_alpha:
            lin("core.%s.alpha_net" % name, 1, A)
    if getattr(opt, "att_input_mode", "both") == "dual_region":        # AttModel.py:126-128, registered after attention2
        lin("core.attention2_dual.h2att", A, H)
        if region_alpha:
            lin("core.attention2_dual.alpha_net", 1, A)
        lin("core.dual_pointer.0", 1, H)
    lin("core.i2h_2", H, 2 * H)
    lin("core.h2h_2", H, H)
    return spec


# multipliers on top of the torch-default init so that greedy captions are not degenerate
# (default init gives 4-6 distinct tokens per batch, SURVEY.md section 7 "hard parts")
_SCALE = {"logit.weight": 10.0, "logit.bias": 0.5, "embed.0.weight": 4.0,
          "core.attention.alpha_net.weight": 8.0, "core.attention2.alpha_net.weight": 8.0,
          "core.attention2_dual.alpha_net.weight": 8.0, "core.dual_pointer.0.weight": 8.0,     # dual_region: the gate spans (0, 1) across clips
          "core.att_lstm.weight_ih": 3.0, "core.lang_lstm.weight_ih": 4.0, "core.lang_lstm.weight_hh": 0.5}
# transformer captioner: sharp attention (so that the caption depends on the clip), a small tied embedding (so that the position, not the
# previous token, dominates the residual stream: with the default init every caption is one token repeated)
for _l in range(2):
    _p = "cap_model.decoder.layers.%d." % _l
    _SCALE.update({_p + "attention.layer.wq.weight": 16.0, _p + "attention.layer.wk.weight": 16.0, _p + "attention.layer.wo.weight": 2.0,
                   _p + "selfattn.layer.wq.weight": 8.0, _p + "selfattn.layer.wk.weight": 8.0,
                   _p + "feedforward.layer.linear2.weight": 2.0})
_SCALE.update({"cap_model.decoder.out.weight": 0.2, "cap_model.decoder.out.bias": 0.2})
# added to logit.bias[UNK] so that UNK is top-1 on a fraction of steps (exercises misc/model.py:590-594)
_UNK_BOOST = 6.0


def make_state_dict(opt, seed=0, scale=None, unk_boost=_UNK_BOOST):
    """Deterministic state_dict with the reference's exact keys/shapes (SURVEY.md 8b)."""
    scale = dict(_SCALE if scale is None else scale)
    sd = {}
    for key, shape, kind, fan in state_dict_spec(opt):
        rs = _rs(seed, key)
        if kind == "uniform":
            k = 1.0 / np.sqrt(fan)
            a = rs.uniform(-k, k, size=shape)
        elif kind == "normal":
            a = rs.standard_normal(shape) / fan
        elif kind == "gamma":
            a = 1.0 + 0.1 * rs.standard_normal(shape)
        elif kind == "var":
            a = rs.uniform(0.5, 1.5, size=shape)
        elif kind == "count":
            sd[key] = torch.tensor(7, dtype=torch.int64)
            continue
        else:
            raise ValueError(kind)
        a = a * scale.get(key, 1.0)
        sd[key] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    sd["logit.bias"][int(opt.wtoi["UNK"])] += unk_boost
    return sd


def make_inputs(opt, B, seed=1234, masked=True, train=False, nbox=3, cap_len=8):
    """Clip tensors as ``main.py:344-350`` (sample) / ``main.py:213-232`` (MLE, GRD) build them.

    masked=True : proposal mask = score <= 0.2 (opts.py:53), masked rows zero-filled
                  (dataloader_anet.py:339-340); masked=False: dense (roofline runs).
    train=True  : also GT boxes copied from proposals (IoU = 1 => non-empty positives),
                  captions with object words, box/frame masks.
    """
    F, T, R = opt.att_feat_size, opt.t_attn_size, opt.num_sampled_frm * opt.num_prop_per_frm
    P, L, V, D = opt.num_prop_per_frm, opt.seq_length, opt.vocab_size, opt.detect_size
    rs = _rs(seed, "inputs")
    out = {}
    out["segs_feat"] = torch.from_numpy(rs.standard_normal((B, T, opt.fc_feat_size)).astype(np.float32))
    feat = np.abs(rs.standard_normal((B, R, F))).astype(np.float32)
    ppls = np.zeros((B, R, 7), dtype=np.float32)
    xy = rs.uniform(0, 300, size=(B, R, 2))
    wh = rs.uniform(1, 300, size=(B, R, 2))
    ppls[:, :, 0:2] = xy
    ppls[:, :, 2:4] = xy + wh
    ppls[:, :, 4] = (np.arange(R) // P)[None, :]
    ppls[:, :, 5] = rs.randint(1, 1601, size=(B, R))
    ppls[:, :, 6] = rs.uniform(0, 1, size=(B, R))
    mask = (ppls[:, :, 6] <= 0.2) if masked else np.zeros((B, R), dtype=bool)
    boxes_at = None
    if train:
        # GT boxes are copies of (unmasked) proposals: proposal 5 of three different frames
        frames = [(k * 4 + 0) % opt.num_sampled_frm for k in range(nbox)]
        boxes_at = np.array([f * P + min(5, P - 1) for f in frames])
        mask[:, boxes_at] = False
    ppls[mask] = 0.0
    feat[mask] = 0.0
    out["ppls"] = torch.from_numpy(ppls)
    out["ppls_feat"] = torch.from_numpy(feat)
    pnt = np.zeros((B, R + 1), dtype=np.uint8)
    pnt[:, 1:] = mask
    out["pnt_mask"] = torch.from_numpy(pnt)
    num = np.zeros((B, 7), dtype=np.int64)
    num[:, 0] = 1
    num[:, 1] = R
    num[:, 2] = nbox if train else 0
    num[:, 3] = rs.randint(0, 6, size=B)
    num[:, 4] = num[:, 3] + rs.randint(1, 6, size=B)
    out["num"] = torch.from_numpy(num)   # int64: start/end fractions truncate to 0 (main.py:572)
    sidx = np.zeros((B, 2), dtype=np.int64)
    for b in range(B):
        lo = (3 * b) % max(1, T // 4)
        hi = T - ((5 * b) % max(1, T // 4))
        sidx[b] = (lo, max(hi, lo + 1))
    out["sample_idx"] = torch.from_numpy(sidx)
    if not train:
        return out

    gt = np.zeros((B, nbox, 6), dtype=np.float32)
    gt[:, :, :5] = ppls[:, boxes_at, :5]
    gt[:, :, 5] = rs.randint(1, D + 1, size=(B, nbox))
    out["gt_boxes"] = torch.from_numpy(gt)
    # frame mask: 1 where proposal and box are on different frames (dataloader_anet.py:168-173)
    frm = (ppls[:, :, 4][:, :, None] != gt[:, :, 4][:, None, :]).astype(np.uint8)
    out["frm_mask"] = torch.from_numpy(frm)
    words = rs.randint(1, V - 1, size=(B, L))
    lens = np.clip(cap_len + rs.randint(-2, 3, size=B), 2 * nbox + 1, L)
    input_seq = np.zeros((B, 1, L + 1, 4), dtype=np.int64)
    gt_seq = np.zeros((B, 10, L), dtype=np.int64)
    box_mask = np.ones((B, 1, nbox, L + 1), dtype=np.uint8)
    for b in range(B):
        n = int(lens[b])
        gt_seq[b, 0, :n] = words[b, :n]
        input_seq[b, 0, 1:n + 1, 0] = words[b, :n]
        for k in range(nbox):
            pos = 2 * k + 1                      # word index of object k
            cls = int(gt[b, k, 5])
            input_seq[b, 0, pos + 1, 0] = V + cls
            input_seq[b, 0, pos + 1, 1] = 1
            input_seq[b, 0, pos + 1, 2] = cls
            input_seq[b, 0, pos + 1, 3] = words[b, pos]
            box_mask[b, 0, k, pos + 1] = 0
    out["input_seq"] = torch.from_numpy(input_seq)
    out["gt_seq"] = torch.from_numpy(gt_seq)
    out["mask_boxes"] = torch.from_numpy(box_mask)
    return out


def make_video_inputs(opt, B, V, seed=1234, masked=True, train=False, nbox=3, cap_len=8):
    """A video-indexed batch: B events of V videos (``TopDownModel.forward(..., eval_opt={'video_idx': ...})``).

    Returns ``make_inputs(opt, B, ...)`` with ``segs_feat`` replaced by V videos' frame features [V, T, F] and a ``video_idx`` [B] (int64;
    every video has an event when B >= V).  The windows ``sample_idx`` cycle through the cases the decode attention treats differently:
    the whole clip, an empty window, one row, a window ending at T, one straddling a temporal chunk boundary, one reaching past T, and
    seeded random windows."""
    T = opt.t_attn_size
    out = make_inputs(opt, B, seed=seed, masked=masked, train=train, nbox=nbox, cap_len=cap_len)
    rs = _rs(seed, "video")
    out["segs_feat"] = torch.from_numpy(rs.standard_normal((V, T, opt.fc_feat_size)).astype(np.float32))
    vid = np.arange(B) % V
    rs.shuffle(vid)
    out["video_idx"] = torch.from_numpy(vid.astype(np.int64))
    mid = max(1, T // 2)
    fixed = [(0, T), (mid, mid), (mid, mid + 1), (max(0, T - 3), T), (max(0, mid - 2), min(T, mid + 2)), (max(0, T - 2), T + 5)]
    sidx = np.zeros((B, 2), dtype=np.int64)
    for b in range(B):
        if b < len(fixed):
            sidx[b] = fixed[b]
        else:
            lo = int(rs.randint(0, T))
            sidx[b] = (lo, int(rs.randint(lo + 1, T + 1)))
    out["sample_idx"] = torch.from_numpy(sidx)
    return out
