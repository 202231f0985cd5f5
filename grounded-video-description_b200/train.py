"""Training step of the top-down captioner on the device (SURVEY.md 8 rows T7 / D1): teacher-forced forward in train mode
(BatchNorm batch statistics; dropout p = 0, see below), the four losses, the explicit backward, global-norm clipping and
per-tensor Adam — `main.py:235-266,660-677` of the reference.

The ORCHESTRATION in this file is verified on the
CPU: `tests/test_train_host_logic.py` runs it with a torch mock of the primitive set (`tests/ops_ref.py`) and compares every
gradient with the oracle (`oracle/gvd_oracle.train_step`, pinned to the reference) — it is a line-by-line transcription of the
verified specification `oracle/gvd_backward.py`.  The PRIMITIVES used by the product (`NativeOps`: csrc/gvd_train.cu through
the C ABI, GEMMs through the wgmma kernel) have their per-primitive tests in
`tests/test_gpu_zz_train.py`.

Dropout: the reference draws its masks from torch's RNG, so bit parity with dropout on is undefined; like the oracle pin this
step runs with every Dropout at p = 0.  (A Philox mask per dropout site is a local change in `lin`/`embed`.)

The primitive set `ops` (all tensors fp32, contiguous, on the device of `ops`):
    lin(x, W, b, relu)              x [..., K] W [N, K] -> [..., N]
    mm_nn(A, B) / mm_tn(A, B)       A [M,N] B [N,K] -> [M,K]   /   A [M,N] B [M,K] -> [N,K]
    bmm_nt / bmm_nn / bmm_tn        batched versions on [b, ., .]
    colsum(x2d), sum_all(x)
    relu_bwd(dy, y), ln / ln_bwd, ln_star / ln_star_bwd, softmax / softmax_bwd
    lstm_cell / lstm_cell_bwd, gru_cell / gru_cell_bwd, att_scores / att_scores_bwd, att_scores_mul / att_scores_mul_bwd, outer_rows
    gather_rows / index_add_rows, lm_nll, pos_nll, cls_nll, bn_train / bn_train_bwd
    add, mul, scale, masked_fill, zeros_like / zeros, cat, clip_adam
"""
import math
import weakref

import torch

try:
    from . import capi
except ImportError:                        # drop-in layout: the package directory itself is on sys.path
    import capi

MIN_VALUE = -1e8


def head_chunks(H, n_heads=6):
    """torch.chunk(n_heads, -1) sizes (transformer.py:121)."""
    c = -(-H // n_heads)
    sizes, left = [], H
    while left > 0:
        sizes.append(min(c, left))
        left -= sizes[-1]
    return sizes


# nn.Dropout / F.dropout sites of the reference's train-mode forward, in execution order (ids key the Philox masks):
#   seg_info (model.py:104-105) fc7 (:158-161) vis_cls (:93-97, the class table of the similarity matrix) loc (:75-77, p = 0.5)
#   pool_embed (:117-119) fc_embed (:99-101) att_rgb / att_mot (:107-112) attn (transformer.py:100, sub = layer*8 + head)
#   res_attn / res_ffn (transformer.py:84-88, sub = layer) gru_l0 (nn.GRU dropout between layers, model.py:153)
#   embed (:79-82, sub = decode step) lang_out (AttModel.py:161, sub = decode step) vis_word (model.py:470, second vis_embed call)
DROP_SITES = {n: i for i, n in enumerate(("seg_info", "fc7", "vis_cls", "loc", "pool_embed", "fc_embed", "att_rgb", "att_mot", "attn", "res_attn",
                                          "res_ffn", "gru_l0", "embed", "lang_out", "vis_word"))}
# The transformer captioner's decoder (att_model = 'transformer'; p = 0.2, model.py:137-142), numbered after the sites above so their masks do
# not change:  tfm_embed (embedding + positional encoding, transformer.py:209)  tfm_attn (attention probabilities, :105,
# sub = (layer * 2 + {0 self, 1 cross}) * 8 + head)  tfm_res (ResidualBlock, :88, sub = layer * 3 + {0 self, 1 cross, 2 feed-forward})
TFM_DROP_SITES = {n: len(DROP_SITES) + i for i, n in enumerate(("tfm_embed", "tfm_attn", "tfm_res"))}
_SITE_IDS = dict(DROP_SITES, **TFM_DROP_SITES)


def check_disable_caption(opt):
    """True when the language loss is part of the objective.  opt.disable_caption (main.py:243-246) drops it; the reference cannot step
    when nothing is left: with w_att2 = w_grd = w_cls = 0 its loss stays the Python int 0 (no .backward()), and the transformer captioner's
    other three losses are constants without a graph (model.py:418-419)."""
    if not getattr(opt, "disable_caption", False):
        return True
    if getattr(opt, "att_model", "topdown") == "transformer":
        raise ValueError("disable_caption with att_model='transformer': the captioner's only loss with a gradient is the language loss")
    if not (opt.w_att2 or opt.w_grd or opt.w_cls):
        raise ValueError("disable_caption with w_att2 = w_grd = w_cls = 0: the training objective is empty")
    return False


class TrainStep:
    """forward_backward(W, opt, inp) -> (losses[4], loss, grads{key});  step(...) adds clip + Adam (first step, main.py:660-677).

    dropout: None (every Dropout at p = 0: the deterministic parity mode the oracle pin uses) or dict(seed=int, p_lm=drop_prob_lm (opts.py: 0.5),
    p_interact=0.2, p_gru=0.2, p_loc=0.5, p_tfm=0.2): train-mode masks at the reference's sites, drawn from counter-based Philox keyed by
    (seed, site, optimisation step) so that the backward regenerates them."""

    def __init__(self, ops, dropout=None):
        self.ops = ops
        self.dropout = dropout
        self.iter = 0

    def _drop(self, x, kind, site, sub, it):
        d = self.dropout
        if not d:
            return x
        p = self._p(kind)
        if p <= 0.0:
            return x
        return self.ops.dropout(x, p, d["seed"], _SITE_IDS[site] * 4096 + sub, it)

    def _p(self, kind):
        d = self.dropout
        if not d:
            return 0.0
        return {"lm": d.get("p_lm", 0.5), "interact": d.get("p_interact", 0.2), "gru": d.get("p_gru", 0.2), "loc": d.get("p_loc", 0.5),
                "tfm": d.get("p_tfm", 0.2)}[kind]

    # ------------------------------------------------------------------ helpers
    def _acc(self, grads, key, g):
        grads[key] = g if key not in grads else self.ops.add(grads[key], g)

    def _lin_bwd(self, dy, x, W, name, grads, need_dx=True):
        ops = self.ops
        dy2, x2 = dy.reshape(-1, dy.shape[-1]), x.reshape(-1, x.shape[-1])
        self._acc(grads, name + ".weight", ops.mm_tn(dy2, x2))
        if (name + ".bias") in W:
            self._acc(grads, name + ".bias", ops.colsum(dy2))
        return ops.mm_nn(dy2, W[name + ".weight"]).reshape(*dy.shape[:-1], x.shape[-1]) if need_dx else None

    def _lstm_fwd(self, x, h, c, W, p):
        ops = self.ops
        gates = ops.add(ops.lin(x, W[p + ".weight_ih"], W[p + ".bias_ih"], False), ops.lin(h, W[p + ".weight_hh"], W[p + ".bias_hh"], False))
        h2, c2, act = ops.lstm_cell(gates, c)
        return h2, c2, dict(act=act, c=c, c2=c2, x=x, h=h)

    def _lstm_bwd(self, dh2, dc2, tp, W, p, grads):
        ops = self.ops
        dgates, dc = ops.lstm_cell_bwd(dh2, dc2, tp["act"], tp["c"], tp["c2"])
        self._acc(grads, p + ".weight_ih", ops.mm_tn(dgates, tp["x"]))
        self._acc(grads, p + ".weight_hh", ops.mm_tn(dgates, tp["h"]))
        bsum = ops.colsum(dgates)
        self._acc(grads, p + ".bias_ih", bsum)
        self._acc(grads, p + ".bias_hh", bsum)
        return ops.mm_nn(dgates, W[p + ".weight_ih"]), ops.mm_nn(dgates, W[p + ".weight_hh"]), dc

    def _attn_fwd(self, p_feats, feats, q, w, b, mask, need_out=True, form="mix"):
        """need_out = False: the scores only (att_input_mode 'featmap' discards the region attention's weighted sum, AttModel.py:145-146).
        form: the score of region_attn_mode (AttModel.py:79-96): 'mix' w . tanh(p + q) + b, 'mix_mul' w . tanh(p * q) + b, 'dp' p . q (w, b
        unused)."""
        ops = self.ops
        if form == "dp":
            s = ops.bmm_nn(p_feats, q.unsqueeze(2)).squeeze(2)                 # [B,N,A] x [B,A,1]
        elif form == "mix_mul":
            s = ops.att_scores_mul(p_feats, q, w, b)
        else:
            s = ops.att_scores(p_feats, q, w, b)
        if mask is not None:
            s = ops.masked_fill(s, mask, MIN_VALUE)
        a = ops.softmax(s, 1.0)
        out = ops.bmm_nn(a.unsqueeze(1), feats).squeeze(1) if need_out else None     # [B,1,N] x [B,N,H]
        return out, s, dict(a=a, mask=mask, q=q, form=form)

    def _attn_bwd(self, dout, ds_extra, tp, p_feats, feats, w, dfeats_acc):
        """dfeats_acc [B,N,H] += a (x) dout in place (the gradient of the attended features, summed over the decode steps).
        dout = None: the weighted sum reached no loss, only the scores did (ds_extra).  Returns (dp_feats, dq, dw, db); dw = db = None in
        the form 'dp' (no alpha_net)."""
        ops = self.ops
        a = tp["a"]
        if dout is None:
            ds = ds_extra
        else:
            ops.outer_rows_acc_(dfeats_acc, a, dout)
            da = ops.bmm_nt(dout.unsqueeze(1), feats).squeeze(1)           # [B,1,H] x [B,N,H]^T -> [B,1,N]
            ds = ops.softmax_bwd(da, a, 1.0)
            if ds_extra is not None:
                ds = ops.add(ds, ds_extra)
        if tp["mask"] is not None:
            ds = ops.masked_fill(ds, tp["mask"], 0.0)
        if tp["form"] == "dp":                                              # s = p . q:  dp = ds (x) q,  dq = sum_n ds p
            return ops.outer_rows(ds, tp["q"]), ops.bmm_nn(ds.unsqueeze(1), p_feats).squeeze(1), None, None
        if tp["form"] == "mix_mul":
            return ops.att_scores_mul_bwd(ds, p_feats, tp["q"], w)
        dpre, dq, dw, db = ops.att_scores_bwd(ds, p_feats, tp["q"], w)
        return dpre, dq, dw, db

    def _gru_dir_fwd(self, x, W, layer, reverse):
        ops = self.ops
        sfx = "_l%d%s" % (layer, "_reverse" if reverse else "")
        Wih, Whh = W["context_enc.weight_ih" + sfx], W["context_enc.weight_hh" + sfx]
        B, T, _ = x.shape
        G = Whh.shape[1]
        gi = ops.lin(x, Wih, W["context_enc.bias_ih" + sfx], False)
        h = ops.zeros((B, G))
        outs = [None] * T
        tape = []
        for t in (range(T - 1, -1, -1) if reverse else range(T)):
            gh = ops.lin(h, Whh, W["context_enc.bias_hh" + sfx], False)
            h2, r, z, n = ops.gru_cell(gi[:, t].contiguous(), gh, h)
            tape.append(dict(t=t, r=r, z=z, n=n, h=h, ghn=gh[:, 2 * G:].contiguous()))
            h = h2
            outs[t] = h
        return ops.stack1(outs), dict(steps=tape, x=x, sfx=sfx, G=G)

    def _gru_dir_bwd(self, dout, tp, W, grads):
        ops = self.ops
        sfx, G, x = tp["sfx"], tp["G"], tp["x"]
        Whh = W["context_enc.weight_hh" + sfx]
        B, T, _ = x.shape
        dgi = [None] * T
        dWhh, dbhh = ops.zeros(tuple(Whh.shape)), ops.zeros((3 * G,))
        dh = ops.zeros((B, G))
        for st in reversed(tp["steps"]):
            t = st["t"]
            dh = ops.add(dh, dout[:, t].contiguous())
            dgi_t, dgh, dh_keep = ops.gru_cell_bwd(dh, st["r"], st["z"], st["n"], st["h"], st["ghn"])
            dgi[t] = dgi_t
            dWhh = ops.add(dWhh, ops.mm_tn(dgh, st["h"]))
            dbhh = ops.add(dbhh, ops.colsum(dgh))
            dh = ops.add(dh_keep, ops.mm_nn(dgh, Whh))
        dgi = ops.stack1(dgi)
        self._acc(grads, "context_enc.weight_hh" + sfx, dWhh)
        self._acc(grads, "context_enc.bias_hh" + sfx, dbhh)
        dgi2 = dgi.reshape(-1, 3 * G)
        self._acc(grads, "context_enc.weight_ih" + sfx, ops.mm_tn(dgi2, x.reshape(-1, x.shape[-1])))
        self._acc(grads, "context_enc.bias_ih" + sfx, ops.colsum(dgi2))
        return ops.mm_nn(dgi2, W["context_enc.weight_ih" + sfx]).reshape(B, T, -1)

    # ------------------------------------------------------------------ prologue (model.py:504-568), shared by both captioners
    def _prologue_fwd(self, W, opt, inp, pmask, keep_d, D_, frames=True, regions=True):
        """Train-mode prologue; returns its tape.  frames / regions = False skips the frame branch / the region branch (the captioner does not
        read it: att_input_mode 'region' / 'featmap' of the transformer, model.py:393)."""
        ops = self.ops
        H = opt.rnn_size
        segs, ppls, num = inp["segs_feat"], inp["ppls"], inp["num"]
        pt = dict(pmask=pmask, segs=segs, fc_feats=None, g_pool=None, simT=None, pool_feats=None, p_pool=None, conv=None, p_conv=None)
        self.last_bn = None
        fc = ops.mean_dim1(segs)
        seg_in = num[:, 3:7].float().contiguous()
        seg_h = D_(ops.lin(seg_in, W["seg_info_embed.0.weight"], W["seg_info_embed.0.bias"], True), "lm", "seg_info")
        ln_fc, ln_seg = ops.ln(fc), ops.ln(seg_h)
        xcat = ops.cat((ln_fc, ln_seg), -1)
        fc_feats = D_(ops.lin(xcat, W["fc_embed.0.weight"], W["fc_embed.0.bias"], True), "lm", "fc_embed")
        pt.update(fc=fc, seg_in=seg_in, seg_h=seg_h, ln_seg=ln_seg, xcat=xcat, fc_feats=fc_feats)

        if regions:
            ppls_feat = inp["ppls_feat"]
            g_pool = D_(ops.lin(ppls_feat, W["ctx2pool_grd.0.weight"], W["ctx2pool_grd.0.bias"], True), "lm", "fc7")
            if getattr(opt, "enable_BUTD", False):
                # BUTD (model.py:357-364): pool_embed reads the dropped-out fc7 output; no similarity, loc_fc, label features or LayerNorms
                Wc = simT = loc_in = loc = ln_g = ln_loc = ln_sim = None
                pool_in = g_pool
            else:
                Wc = D_(ops.relu(W["vis_embed.0.weight"]), "lm", "vis_cls")                 # ONE mask for the class table (model.py:320-321)
                simT_raw = ops.lin(g_pool, Wc, W.get("vis_classifiers_bias"), False)         # B, R, C (region-major); no bias in transfer_mode 'none'
                simT_raw = ops.masked_fill(simT_raw, pmask.unsqueeze(-1).expand_as(simT_raw), MIN_VALUE)
                simT = ops.softmax(simT_raw, 1.0)                                            # softmax over the classes

                loc_in = ops.cat((ops.scale(ppls[:, :, :4].contiguous(), 1.0 / 720.0), ops.scale(ppls[:, :, 4:5].contiguous(), 1.0 / float(opt.num_sampled_frm))), -1)
                loc = D_(ops.lin(loc_in, W["loc_fc.0.weight"], W["loc_fc.0.bias"], True), "loc", "loc")
                ln_g, ln_loc, ln_sim = ops.ln(g_pool), ops.ln(loc), ops.ln(simT)
                pool_in = ops.cat((ln_g, ln_loc, ln_sim), -1)
            pool_embed = D_(ops.lin(pool_in, W["pool_embed.0.weight"], W["pool_embed.0.bias"], True), "lm", "pool_embed")
            pool = pool_embed

            it_tape = []
            if opt.obj_interact:
                sizes = head_chunks(H)
                scale = 1.0 / math.sqrt(H)
                x = pool
                for l in range(2):
                    p = "obj_interact.encoder.layers.%d." % l
                    q = ops.lin(x, W[p + "selfattn.layer.wq.weight"], None, False)
                    k = ops.lin(x, W[p + "selfattn.layer.wk.weight"], None, False)
                    v = ops.lin(x, W[p + "selfattn.layer.wv.weight"], None, False)
                    heads, outs, o = [], [], 0
                    for hi, s in enumerate(sizes):
                        qh, kh, vh = (t[..., o:o + s].contiguous() for t in (q, k, v))
                        att = ops.softmax(ops.bmm_nt(qh, kh), scale)
                        att_d = D_(att, "interact", "attn", l * 8 + hi)                     # transformer.py:100
                        outs.append(ops.bmm_nn(att_d, vh))
                        heads.append((att, qh, kh, vh, att_d))
                        o += s
                    cat = ops.cat(outs, -1)
                    a = D_(ops.lin(cat, W[p + "selfattn.layer.wo.weight"], None, False), "interact", "res_attn", l)     # transformer.py:88
                    x1_in = ops.add(x, a)
                    x1 = ops.ln_star(x1_in, W[p + "selfattn.layernorm.gamma"], W[p + "selfattn.layernorm.beta"])
                    f1 = ops.lin(x1, W[p + "feedforward.layer.linear1.weight"], W[p + "feedforward.layer.linear1.bias"], True)
                    f2 = D_(ops.lin(f1, W[p + "feedforward.layer.linear2.weight"], W[p + "feedforward.layer.linear2.bias"], False), "interact", "res_ffn", l)
                    x2_in = ops.add(x1, f2)
                    x2 = ops.ln_star(x2_in, W[p + "feedforward.layernorm.gamma"], W[p + "feedforward.layernorm.beta"])
                    it_tape.append(dict(l=l, p=p, x=x, heads=heads, cat=cat, x1_in=x1_in, x1=x1, f1=f1, x2_in=x2_in))
                    x = x2
                pool = x
            pool_feats = pool
            p_pool = ops.lin(pool_feats, W["ctx2pool.weight"], W["ctx2pool.bias"], False)
            pt.update(ppls_feat=ppls_feat, g_pool=g_pool, Wc=Wc, simT=simT, loc_in=loc_in, loc=loc, ln_g=ln_g, ln_loc=ln_loc, ln_sim=ln_sim,
                      pool_in=pool_in, pool_embed=pool_embed, it_tape=it_tape, pool_feats=pool_feats, p_pool=p_pool)

        if frames:
            e_rgb = D_(ops.lin(segs[..., :2048].contiguous(), W["att_embed.0.0.weight"], W["att_embed.0.0.bias"], True), "lm", "att_rgb")
            e_mot = D_(ops.lin(segs[..., 2048:].contiguous(), W["att_embed.1.0.weight"], W["att_embed.1.0.bias"], True), "lm", "att_mot")
            e = ops.cat((e_rgb, e_mot), -1)
            bn = "att_embed_aux.0."
            Bt, T = e.shape[0], e.shape[1]
            e2 = e.reshape(Bt * T, -1)
            e_hat, bn_var = ops.bn_train(e2)                                                # statistics of this batch (train mode)
            self.last_bn = (ops.scale(ops.colsum(e2), 1.0 / (Bt * T)), bn_var, Bt * T)       # batch mean / biased variance / count: running-stat update
            e_bn = ops.add(ops.mul(e_hat, W[bn + "weight"].unsqueeze(0).expand_as(e_hat).contiguous()), W[bn + "bias"].unsqueeze(0).expand_as(e_hat).contiguous())
            gx = ops.relu(e_bn).reshape(Bt, T, -1)
            gru_tapes, gin = [], gx
            for layer in range(2):
                of, tf = self._gru_dir_fwd(gin, W, layer, False)
                ob, tb = self._gru_dir_fwd(gin, W, layer, True)
                gru_tapes.append((tf, tb))
                gin = ops.cat((of, ob), -1)
                if layer == 0:
                    gin = D_(gin, "gru", "gru_l0")                                            # nn.GRU(dropout=0.2): between the layers only
            keep = keep_d.expand(Bt, T, gin.shape[-1]).contiguous()
            conv = ops.mul(gin, keep)
            p_conv = ops.lin(conv, W["ctx2att.weight"], W["ctx2att.bias"], False)
            pt.update(e_rgb=e_rgb, e_mot=e_mot, e_hat=e_hat, bn_var=bn_var, e_bn=e_bn, gru_tapes=gru_tapes, keep=keep, conv=conv, p_conv=p_conv)
        return pt

    def _prologue_bwd(self, pt, W, opt, grads, D_, dconv=None, dp_conv=None, dfc_feats=None, dpool_feats=None, dp_pool=None, dg_pool=None, dsimT=None):
        """Backward of _prologue_fwd for the gradients of its outputs (None = the captioner did not read that output: its parameters get no
        gradient).  Accumulates into `grads`."""
        ops = self.ops
        H = opt.rnn_size
        if dp_conv is not None:
            dconv = ops.add(dconv, self._lin_bwd(dp_conv, pt["conv"], W, "ctx2att", grads))
        if dconv is not None:
            e_bn, e_hat, e_rgb, e_mot, segs, bn = pt["e_bn"], pt["e_hat"], pt["e_rgb"], pt["e_mot"], pt["segs"], "att_embed_aux.0."
            Bt, T = e_rgb.shape[0], e_rgb.shape[1]
            dgin = ops.mul(dconv, pt["keep"])
            G = dgin.shape[-1] // 2
            for layer in (1, 0):
                tf, tb = pt["gru_tapes"][layer]
                if layer == 0:
                    dgin = D_(dgin, "gru", "gru_l0")
                dgin = ops.add(self._gru_dir_bwd(dgin[..., :G].contiguous(), tf, W, grads), self._gru_dir_bwd(dgin[..., G:].contiguous(), tb, W, grads))
            de_bn = ops.relu_bwd(dgin.reshape(Bt * T, -1), e_bn)
            self._acc(grads, bn + "weight", ops.colsum(ops.mul(de_bn, e_hat)))
            self._acc(grads, bn + "bias", ops.colsum(de_bn))
            dxh = ops.mul(de_bn, W[bn + "weight"].unsqueeze(0).expand_as(de_bn).contiguous())
            de = ops.bn_train_bwd(dxh, e_hat, pt["bn_var"]).reshape(Bt, T, -1)
            Hh = e_rgb.shape[-1]
            de_rgb = ops.relu_bwd(D_(de[..., :Hh].contiguous(), "lm", "att_rgb"), e_rgb)
            de_mot = ops.relu_bwd(D_(de[..., Hh:].contiguous(), "lm", "att_mot"), e_mot)
            self._lin_bwd(de_rgb, segs[..., :2048].contiguous(), W, "att_embed.0.0", grads, need_dx=False)
            self._lin_bwd(de_mot, segs[..., 2048:].contiguous(), W, "att_embed.1.0", grads, need_dx=False)

        if dfc_feats is not None:
            fc_feats, seg_h = pt["fc_feats"], pt["seg_h"]
            dxcat = self._lin_bwd(ops.relu_bwd(D_(dfc_feats, "lm", "fc_embed"), fc_feats), pt["xcat"], W, "fc_embed.0", grads)
            dseg_h = ops.relu_bwd(D_(ops.ln_bwd(dxcat[:, pt["fc"].shape[1]:].contiguous(), pt["ln_seg"], seg_h), "lm", "seg_info"), seg_h)
            self._lin_bwd(dseg_h, pt["seg_in"], W, "seg_info_embed.0", grads, need_dx=False)

        if dpool_feats is None and dsimT is None:
            return
        g_pool, simT, pmask = pt["g_pool"], pt["simT"], pt["pmask"]
        if dpool_feats is not None:
            dg_pool, dsimT = self._pool_bwd(pt, W, opt, grads, D_, dpool_feats, dp_pool, dg_pool, dsimT)
        if dsimT is not None:                            # (BUTD: no similarity, so vis_embed and the class bias get no gradient)
            n_g = g_pool.shape[-1]
            dsim_raw = ops.masked_fill(ops.softmax_bwd(dsimT, simT, 1.0), pmask.unsqueeze(-1).expand_as(simT), 0.0)  # B, R, C
            dsr2, gp2 = dsim_raw.reshape(-1, dsim_raw.shape[-1]), g_pool.reshape(-1, n_g)
            dg_sim = ops.mm_nn(dsr2, pt["Wc"]).reshape(tuple(g_pool.shape))
            dg_pool = dg_sim if dg_pool is None else ops.add(dg_pool, dg_sim)
            self._acc(grads, "vis_embed.0.weight", ops.relu_bwd(D_(ops.mm_tn(dsr2, gp2), "lm", "vis_cls"), W["vis_embed.0.weight"]))
            if "vis_classifiers_bias" in W:
                self._acc(grads, "vis_classifiers_bias", ops.colsum(dsr2))
        self._lin_bwd(ops.relu_bwd(D_(dg_pool, "lm", "fc7"), g_pool), pt["ppls_feat"], W, "ctx2pool_grd.0", grads, need_dx=False)

    def _pool_bwd(self, pt, W, opt, grads, D_, dpool_feats, dp_pool, dg_pool, dsimT):
        """Backward of the region features (ctx2pool, obj_interact, pool_embed, loc_fc) into the gradients of g_pool and of the similarity."""
        ops = self.ops
        H = opt.rnn_size
        pool_feats, g_pool, simT, loc = pt["pool_feats"], pt["g_pool"], pt["simT"], pt["loc"]
        dpool = ops.add(dpool_feats, self._lin_bwd(dp_pool, pool_feats, W, "ctx2pool", grads)) if dp_pool is not None else dpool_feats
        if opt.obj_interact:
            sizes = head_chunks(H)
            scale = 1.0 / math.sqrt(H)
            for tp in reversed(pt["it_tape"]):
                p = tp["p"]
                dx2_in, dg_, db_ = ops.ln_star_bwd(dpool, tp["x2_in"], W[p + "feedforward.layernorm.gamma"])
                self._acc(grads, p + "feedforward.layernorm.gamma", dg_)
                self._acc(grads, p + "feedforward.layernorm.beta", db_)
                df1 = ops.relu_bwd(self._lin_bwd(D_(dx2_in, "interact", "res_ffn", tp["l"]), tp["f1"], W, p + "feedforward.layer.linear2", grads), tp["f1"])
                dx1 = ops.add(dx2_in, self._lin_bwd(df1, tp["x1"], W, p + "feedforward.layer.linear1", grads))
                dx1_in, dg_, db_ = ops.ln_star_bwd(dx1, tp["x1_in"], W[p + "selfattn.layernorm.gamma"])
                self._acc(grads, p + "selfattn.layernorm.gamma", dg_)
                self._acc(grads, p + "selfattn.layernorm.beta", db_)
                dcat = self._lin_bwd(D_(dx1_in, "interact", "res_attn", tp["l"]), tp["cat"], W, p + "selfattn.layer.wo", grads)
                dqs, dks, dvs, o = [], [], [], 0
                for hi, (s, (att, qh, kh, vh, att_d)) in enumerate(zip(sizes, tp["heads"])):
                    do = dcat[..., o:o + s].contiguous()
                    dvs.append(ops.bmm_tn(att_d, do))                                    # (dropped att)^T do
                    dsc = ops.softmax_bwd(D_(ops.bmm_nt(do, vh), "interact", "attn", tp["l"] * 8 + hi), att, scale)
                    dqs.append(ops.bmm_nn(dsc, kh))
                    dks.append(ops.bmm_tn(dsc, qh))
                    o += s
                dx = dx1_in
                for nm, parts in (("wq", dqs), ("wk", dks), ("wv", dvs)):
                    dx = ops.add(dx, self._lin_bwd(ops.cat(parts, -1), tp["x"], W, p + "selfattn.layer.%s" % nm, grads))
                dpool = dx
        dpool_in = self._lin_bwd(ops.relu_bwd(D_(dpool, "lm", "pool_embed"), pt["pool_embed"]), pt["pool_in"], W, "pool_embed.0", grads)
        if getattr(opt, "enable_BUTD", False):            # pool_embed read fc7 directly: its input gradient is fc7's (model.py:357-364)
            return dpool_in if dg_pool is None else ops.add(dg_pool, dpool_in), dsimT
        n_g, n_l = g_pool.shape[-1], loc.shape[-1]
        dg_ln = ops.ln_bwd(dpool_in[..., :n_g].contiguous(), pt["ln_g"], g_pool)
        dg_pool = dg_ln if dg_pool is None else ops.add(dg_pool, dg_ln)
        dloc = ops.relu_bwd(D_(ops.ln_bwd(dpool_in[..., n_g:n_g + n_l].contiguous(), pt["ln_loc"], loc), "loc", "loc"), loc)
        self._lin_bwd(dloc, pt["loc_in"], W, "loc_fc.0", grads, need_dx=False)
        dsim_ln = ops.ln_bwd(dpool_in[..., n_g + n_l:].contiguous(), pt["ln_sim"], simT)
        dsimT = dsim_ln if dsimT is None else ops.add(dsimT, dsim_ln)
        return dg_pool, dsimT

    # ------------------------------------------------------------------ the step
    def forward(self, W, opt, inp, host=None):
        """Teacher-forced forward in train mode; returns (the four losses, backward) where backward(w_lm, w_att2, w_grd, w_cls)
        runs the explicit backward for the given loss weights.  `inp` tensors on the device of `ops`; `host` = the CPU copies of the integer / mask inputs that drive control flow
        (targets of the teacher forcing, the early exit `seq[:, i].sum() == 0`, model.py:425) — defaults to `inp`."""
        if getattr(opt, "att_model", "topdown") == "transformer":
            return self._tfm_forward(W, opt, inp, host)
        ops = self.ops
        host = host or inp
        it = self.iter                                                                  # keys this step's dropout masks (forward AND backward)
        self.iter += 1
        D_ = lambda x, kind, site, sub=0: self._drop(x, kind, site, sub, it)
        B = inp["ppls"].shape[0]
        H, L, V = opt.rnn_size, opt.seq_length, opt.vocab_size
        pnt_mask = inp["pnt_mask"]
        pmask = pnt_mask[:, 1:].bool()
        # ---- everything the control flow derives from the host copies of the integer inputs, uploaded in ONE burst before any kernel of the
        # step is queued (a pageable host-to-device copy in the middle of the step would drain the stream every time)
        seq_h = torch.cat((torch.zeros(B, 1, dtype=torch.long), host["gt_seq"][:, 0, :].cpu()), dim=1)
        S = 1
        while S < L and int(seq_h[:, S].sum()) != 0:                                     # model.py:425: stop at the first all-zero column
            S += 1
        T_ = inp["segs_feat"].shape[1]
        sidx = host["sample_idx"].cpu()
        tt = torch.arange(T_).view(1, T_)
        keep_h = ((tt >= sidx[:, 0:1]) & (tt < sidx[:, 1:2])).unsqueeze(-1).float()
        txt_mask_h = torch.cat((torch.ones(B, 1, dtype=torch.bool), seq_h[:, 1:S] > 0), dim=1)
        cls_idx_h = (host["input_seq"][:, 0, 1:S + 1, 0].cpu() - V).clamp(min=0)
        seq_d = ops.to_device(seq_h.t().contiguous())                                    # [L+1, B]: row i = the tokens fed at step i
        keep_d = ops.to_device(keep_h.contiguous())                                      # [B, T, 1]
        txt_mask_d = ops.to_device(txt_mask_h)
        cls_idx = ops.to_device(cls_idx_h.reshape(-1).contiguous())

        mode = getattr(opt, "att_input_mode", "both")
        featmap = mode == "featmap"                     # language LSTM input cat(att, h_att) (AttModel.py:145-146)
        dual = mode == "dual_region"                    # cat(g att2 + (1 - g) att2_dual, h_att), no frame branch (AttModel.py:153-156, model.py:393)
        form = getattr(opt, "region_attn_mode", "mix")  # the region attentions' score (AttModel.py:79-96); the temporal one is additive
        pt = self._prologue_fwd(W, opt, inp, pmask, keep_d, D_, frames=not dual)
        fc_feats, g_pool, simT, pool_feats, p_pool, conv, p_conv = (pt[k] for k in ("fc_feats", "g_pool", "simT", "pool_feats", "p_pool", "conv",
                                                                                      "p_conv"))

        # ========================================================== forward, teacher-forced loop
        tgt = ops.host_targets(self, opt, inp, host)                                     # overlaps, class targets, per-step labels / masks
        a1w, a1b = W["core.attention.alpha_net.weight"], W["core.attention.alpha_net.bias"]
        a2w, a2b = W.get("core.attention2.alpha_net.weight"), W.get("core.attention2.alpha_net.bias")          # (None in 'dp')
        if dual:
            adw, adb = W.get("core.attention2_dual.alpha_net.weight"), W.get("core.attention2_dual.alpha_net.bias")
        h_att = c_att = h_lang = c_lang = ops.zeros((B, H))
        steps, outs, z_list = [], [], []
        for i in range(S):                                                               # S: the reference's early exit (model.py:425)
            tok = seq_d[i]
            emb_raw = ops.gather_rows(W["embed.0.weight"], tok)
            xt = D_(ops.relu(emb_raw), "lm", "embed", i)
            x_att = ops.cat((fc_feats, xt), 1)
            h_att2, c_att2, t_att = self._lstm_fwd(x_att, h_att, c_att, W, "core.att_lstm")
            if not dual:
                q1 = ops.lin(h_att2, W["core.attention.h2att.weight"], W["core.attention.h2att.bias"], False)
                att, _, t_a1 = self._attn_fwd(p_conv, conv, q1, a1w, a1b, None)
            q2 = ops.lin(h_att2, W["core.attention2.h2att.weight"], W["core.attention2.h2att.bias"], False)
            att2, z, t_a2 = self._attn_fwd(p_pool, pool_feats, q2, a2w, a2b, pmask, need_out=not featmap, form=form)
            fmask = tgt["fm"][i]                                                         # B, R (bool): frame mask | proposal mask
            z_out = ops.masked_fill(z, fmask, MIN_VALUE)
            st = dict(tok=tok, emb_raw=emb_raw, t_att=t_att, t_a2=t_a2, h_att2=h_att2, fmask=fmask)
            if dual:
                qd = ops.lin(h_att2, W["core.attention2_dual.h2att.weight"], W["core.attention2_dual.h2att.bias"], False)
                att2d, _, t_ad = self._attn_fwd(p_pool, pool_feats, qd, adw, adb, pmask, form=form)
                # g = sigmoid(dual_pointer(h_att)) as column 0 of softmax([logit, 0]); column 1 is 1 - g
                # (the single-output Linear as a row dot product: no GEMM with one output column)
                wpE = W["core.dual_pointer.0.weight"].expand(B, H).contiguous()
                glog = ops.add(ops.rowsum(ops.mul(h_att2, wpE)).reshape(B, 1), W["core.dual_pointer.0.bias"].reshape(1, 1).expand(B, 1).contiguous())
                gp = ops.softmax(ops.cat((glog, ops.zeros((B, 1))), 1), 1.0)
                gE, hE = (gp[:, k:k + 1].expand(B, H).contiguous() for k in (0, 1))
                x_lang = ops.cat((ops.add(ops.mul(gE, att2), ops.mul(hE, att2d)), h_att2), 1)
                st.update(t_ad=t_ad, att2=att2, att2d=att2d, gp=gp, gE=gE, hE=hE, wpE=wpE)
            else:
                x_lang = ops.cat((att if featmap else ops.add(att, att2), h_att2), 1)
                st.update(t_a1=t_a1)
            h_lang2, c_lang2, t_lang = self._lstm_fwd(x_lang, h_lang, c_lang, W, "core.lang_lstm")
            st.update(t_lang=t_lang)
            steps.append(st)
            outs.append(D_(h_lang2, "lm", "lang_out", i))                                  # AttModel.py:161: the state keeps the un-dropped h
            z_list.append(z_out)
            h_att, c_att, h_lang, c_lang = h_att2, c_att2, h_lang2, c_lang2
        outs_t = ops.stack1(outs)                                                        # B, S, H
        logits = ops.lin(outs_t, W["logit.weight"], W["logit.bias"], False)
        z_all = ops.stack1(z_list)                                                       # B, S, R
        target = seq_d[1:S + 1].t().contiguous()
        lm, dlogits = ops.lm_nll(logits, target, txt_mask_d)                             # dlogits for d(lm) = 1
        pos = tgt["labels"][:, :S].contiguous()                                          # B, S, R (bool)
        gmask = tgt["fm_all"][:, :S].contiguous()
        emb_cls_raw = ops.gather_rows(W["vis_embed.0.weight"], cls_idx).reshape(B, S, -1)
        emb_cls = D_(ops.relu(emb_cls_raw), "lm", "vis_word")
        cls_bias = W.get("vis_classifiers_bias")                                         # None in transfer_mode 'none' (model.py:472-476)
        grd = ops.bmm_nt(emb_cls, g_pool)
        if cls_bias is not None:
            grd = ops.add(grd, ops.gather_rows(cls_bias.unsqueeze(1).contiguous(), cls_idx).reshape(B, S, 1).expand(B, S, z_all.shape[-1]).contiguous())
        grd = ops.add(grd, z_all)
        grd = ops.masked_fill(grd, gmask, MIN_VALUE)
        att2_loss, dz_unit = ops.pos_nll(z_all, pos)
        grd_loss, dgrd_unit = ops.pos_nll(grd, pos)
        cls_loss, dsimT_unit = ops.cls_nll(simT, tgt["cls_target"])                      # on the region-major similarity
        def backward(w_lm, w_att2, w_grd, w_cls):
            """Explicit backward of  w_lm lm + w_att2 att2 + w_grd grd + w_cls cls  (weights = the upstream gradients of the four
            losses): one pass, linear in the weights.  Returns {parameter key: gradient}."""
            grads = {}
            # featmap: the region attention reaches the loss through its logits only, so with w_att2 = w_grd = 0 the region branch gets no
            # gradient at all (None in the reference: Adam skips it)
            region_grad = not featmap or bool(w_att2) or bool(w_grd)
            # ========================================================== backward, loss heads
            # w_lm = 0 (disable_caption, main.py:243-246): the logit head gets no gradient (None in the reference).  Everything else still
            # gets one, exact zeros where only the language loss reached it: the reference's decode state is torch.stack([h_att, h_lang])
            # (AttModel.py:163), so the next step's h_att = state[0][0] carries a zero gradient into h_lang, the language LSTM and its inputs.
            douts = self._lin_bwd(ops.scale(dlogits, w_lm), outs_t, W, "logit", grads) if w_lm else ops.zeros(tuple(outs_t.shape))
            dz_all = ops.zeros(tuple(z_all.shape))
            dg_pool = ops.zeros(tuple(g_pool.shape))
            if w_att2:
                dz_all = ops.add(dz_all, ops.scale(dz_unit, w_att2))
            if w_grd:
                dgrd = ops.masked_fill(ops.scale(dgrd_unit, w_grd), gmask, 0.0)
                dz_all = ops.add(dz_all, dgrd)
                dg_pool = ops.add(dg_pool, ops.bmm_tn(dgrd, emb_cls))                        # [B,S,R]^T [B,S,D] -> [B,R,D]
                demb = ops.relu_bwd(D_(ops.bmm_nn(dgrd, g_pool), "lm", "vis_word"), emb_cls_raw)   # [B,S,R] [B,R,D] -> [B,S,D]
                self._acc(grads, "vis_embed.0.weight", ops.index_add_rows(W["vis_embed.0.weight"].shape[0], cls_idx, demb.reshape(B * S, -1)))
                if cls_bias is not None:
                    self._acc(grads, "vis_classifiers_bias", ops.index_add_rows(cls_bias.shape[0], cls_idx, ops.rowsum(dgrd.reshape(B * S, -1)).reshape(-1, 1)).reshape(-1))
            dsimT = ops.scale(dsimT_unit, w_cls) if w_cls else (ops.zeros(tuple(simT.shape)) if region_grad else None)

            # ========================================================== backward, BPTT over the decode steps
            dp_pool, dpool_feats = ops.zeros(tuple(p_pool.shape)), ops.zeros(tuple(pool_feats.shape))
            dp_conv, dconv = (None, None) if dual else (ops.zeros(tuple(p_conv.shape)), ops.zeros(tuple(conv.shape)))
            dfc_feats = ops.zeros(tuple(fc_feats.shape))
            E = W["embed.0.weight"].shape[1]
            dembed = ops.zeros(tuple(W["embed.0.weight"].shape))
            zBH = ops.zeros((B, H))
            dh_att_n = dc_att_n = dh_lang_n = dc_lang_n = zBH
            for i in range(S - 1, -1, -1):
                st = steps[i]
                dx_lang, dh_lang_n, dc_lang_n = self._lstm_bwd(ops.add(D_(douts[:, i].contiguous(), "lm", "lang_out", i), dh_lang_n), dc_lang_n, st["t_lang"], W,
                                                               "core.lang_lstm", grads)
                datt_sum = dx_lang[:, :H].contiguous()
                dh_att = ops.add(dx_lang[:, H:].contiguous(), dh_att_n)
                datt2 = datt_sum
                if dual:
                    # x = g att2 + (1 - g) att2_dual: d att2 = g dx, d att2_dual = (1 - g) dx, d logit = g (1 - g) sum_h dx (att2 - att2_dual)
                    datt2 = ops.mul(st["gE"], datt_sum)
                    dgd = ops.mul(st["hE"], datt_sum)
                    dg = ops.rowsum(ops.mul(datt_sum, ops.add(st["att2"], ops.scale(st["att2d"], -1.0)))).reshape(B, 1)
                    gp = st["gp"]
                    dglog = ops.mul(dg, ops.mul(gp[:, 0:1].contiguous(), gp[:, 1:2].contiguous()))
                    dglogE = dglog.expand(B, H).contiguous()
                    self._acc(grads, "core.dual_pointer.0.weight", ops.colsum(ops.mul(dglogE, st["h_att2"])).reshape(1, H))
                    self._acc(grads, "core.dual_pointer.0.bias", ops.sum_all(dglog))
                    dh_att = ops.add(dh_att, ops.mul(dglogE, st["wpE"]))
                    dpd, dqd, dwd, dbd = self._attn_bwd(dgd, None, st["t_ad"], p_pool, pool_feats, adw, dpool_feats)
                    dp_pool = ops.add(dp_pool, dpd)
                    if dwd is not None:
                        self._acc(grads, "core.attention2_dual.alpha_net.weight", dwd.reshape(1, -1))
                        self._acc(grads, "core.attention2_dual.alpha_net.bias", dbd.reshape(1))
                    dh_att = ops.add(dh_att, self._lin_bwd(dqd, st["h_att2"], W, "core.attention2_dual.h2att", grads))
                if region_grad:
                    dz = ops.masked_fill(dz_all[:, i].contiguous(), st["fmask"], 0.0)
                    dpp, dq2, dw2, db2 = self._attn_bwd(None if featmap else datt2, dz, st["t_a2"], p_pool, pool_feats, a2w, dpool_feats)
                    dp_pool = ops.add(dp_pool, dpp)
                    if dw2 is not None:
                        self._acc(grads, "core.attention2.alpha_net.weight", dw2.reshape(1, -1))
                        self._acc(grads, "core.attention2.alpha_net.bias", db2.reshape(1))
                    dh_att = ops.add(dh_att, self._lin_bwd(dq2, st["h_att2"], W, "core.attention2.h2att", grads))
                if not dual:
                    dpc, dq1, dw1, db1 = self._attn_bwd(datt_sum, None, st["t_a1"], p_conv, conv, a1w, dconv)
                    dp_conv = ops.add(dp_conv, dpc)
                    self._acc(grads, "core.attention.alpha_net.weight", dw1.reshape(1, -1))
                    self._acc(grads, "core.attention.alpha_net.bias", db1.reshape(1))
                    dh_att = ops.add(dh_att, self._lin_bwd(dq1, st["h_att2"], W, "core.attention.h2att", grads))
                dx_att, dh_att_n, dc_att_n = self._lstm_bwd(dh_att, dc_att_n, st["t_att"], W, "core.att_lstm", grads)
                dfc_feats = ops.add(dfc_feats, dx_att[:, :H].contiguous())
                dembed = ops.add(dembed, ops.index_add_rows(dembed.shape[0], st["tok"], ops.relu_bwd(D_(dx_att[:, H:H + E].contiguous(), "lm", "embed", i), st["emb_raw"])))
            self._acc(grads, "embed.0.weight", dembed)

            if not region_grad:
                dpool_feats = dp_pool = dg_pool = None
            self._prologue_bwd(pt, W, opt, grads, D_, dconv=dconv, dp_conv=dp_conv, dfc_feats=dfc_feats, dpool_feats=dpool_feats, dp_pool=dp_pool,
                               dg_pool=dg_pool, dsimT=dsimT)
            return grads

        return [lm, att2_loss, grd_loss, cls_loss], backward

    def _tfm_forward(self, W, opt, inp, host=None):
        """att_model = 'transformer' (model.py:404-419): the train-mode prologue, then the teacher-forced decoder of TransformerDecoder.forward
        (transformer.py:207-212,276-283) over seq = [0, gt_seq][:, :-1] and F.cross_entropy over the positions whose target is non-zero.  Returns
        ([lm, 0, 0, 0], backward) like forward(): the captioner has no box supervision, so only w_lm is read."""
        ops = self.ops
        host = host or inp
        it = self.iter
        self.iter += 1
        D_ = lambda x, kind, site, sub=0: self._drop(x, kind, site, sub, it)
        B = inp["ppls"].shape[0]
        H, L, V = opt.rnn_size, opt.seq_length, opt.vocab_size
        mode = opt.att_input_mode
        if mode not in ("both", "featmap", "region"):
            raise NotImplementedError(mode)
        seq_h = torch.cat((torch.zeros(B, 1, dtype=torch.long), host["gt_seq"][:, 0, :].cpu().long()), dim=1)       # model.py:285-286
        if int(seq_h.min()) < 0 or int(seq_h.max()) >= V:
            raise IndexError("caption token id outside [0, %d)" % V)
        s_in_h, tgt_h = seq_h[:, :-1].contiguous(), seq_h[:, 1:].contiguous()
        keep_tok_h = tgt_h != 0
        if not bool(keep_tok_h.any()):
            # the reference's cross_entropy over no position is NaN and Adam would write NaN into every weight
            raise capi.GvdError("no caption position has a non-zero target: the language loss is a mean over nothing")
        T_ = inp["segs_feat"].shape[1]
        sidx = host["sample_idx"].cpu()
        tt = torch.arange(T_).view(1, T_)
        keep_h = ((tt >= sidx[:, 0:1]) & (tt < sidx[:, 1:2])).unsqueeze(-1).float()
        pe_h = capi.positional_encodings(L, H).unsqueeze(0).expand(B, L, H).contiguous()
        s_in = ops.to_device(s_in_h.reshape(-1))                                           # one upload burst before any kernel of the step
        tgt = ops.to_device(tgt_h)
        keep_tok = ops.to_device(keep_tok_h)
        keep_d = ops.to_device(keep_h.contiguous())
        pe = ops.to_device(pe_h)

        frames, regions = mode != "region", mode != "featmap"
        pt = self._prologue_fwd(W, opt, inp, inp["pnt_mask"][:, 1:].bool(), keep_d, D_, frames=frames, regions=regions)
        enc = {"both": ("conv", "pool_feats"), "featmap": ("conv", "conv"), "region": ("pool_feats", "pool_feats")}[mode]

        scale = 1.0 / math.sqrt(H)
        p_att = self._p("tfm")
        seed = self.dropout["seed"] if self.dropout else 0
        site = lambda l, cross: _SITE_IDS["tfm_attn"] * 4096 + (l * 2 + cross) * 8
        dec = "cap_model.decoder."
        emb_raw = ops.gather_rows(W[dec + "out.weight"], s_in).reshape(B, L, H)
        x = D_(ops.add(ops.scale(emb_raw, math.sqrt(H)), pe), "tfm", "tfm_embed")              # F.embedding(x, out.weight * sqrt(d)) + pe
        tape = []
        for l in range(2):
            p = dec + "layers.%d." % l
            e = pt[enc[l]]
            q = ops.lin(x, W[p + "selfattn.layer.wq.weight"], None, False)
            k = ops.lin(x, W[p + "selfattn.layer.wk.weight"], None, False)
            v = ops.lin(x, W[p + "selfattn.layer.wv.weight"], None, False)
            a, lse = ops.mha_fwd(q, k, v, True, scale, p_att, seed, site(l, 0), it)
            x1_in = ops.add(x, D_(ops.lin(a, W[p + "selfattn.layer.wo.weight"], None, False), "tfm", "tfm_res", l * 3))
            x1 = ops.ln_star(x1_in, W[p + "selfattn.layernorm.gamma"], W[p + "selfattn.layernorm.beta"])
            q2 = ops.lin(x1, W[p + "attention.layer.wq.weight"], None, False)
            k2 = ops.lin(e, W[p + "attention.layer.wk.weight"], None, False)
            v2 = ops.lin(e, W[p + "attention.layer.wv.weight"], None, False)
            c, lse2 = ops.mha_fwd(q2, k2, v2, False, scale, p_att, seed, site(l, 1), it)
            x2_in = ops.add(x1, D_(ops.lin(c, W[p + "attention.layer.wo.weight"], None, False), "tfm", "tfm_res", l * 3 + 1))
            x2 = ops.ln_star(x2_in, W[p + "attention.layernorm.gamma"], W[p + "attention.layernorm.beta"])
            f1 = ops.lin(x2, W[p + "feedforward.layer.linear1.weight"], W[p + "feedforward.layer.linear1.bias"], True)
            f2 = D_(ops.lin(f1, W[p + "feedforward.layer.linear2.weight"], W[p + "feedforward.layer.linear2.bias"], False), "tfm", "tfm_res", l * 3 + 2)
            x3_in = ops.add(x2, f2)
            tape.append(dict(p=p, e=e, x=x, q=q, k=k, v=v, a=a, lse=lse, x1_in=x1_in, x1=x1, q2=q2, k2=k2, v2=v2, c=c, lse2=lse2, x2_in=x2_in,
                             x2=x2, f1=f1, x3_in=x3_in))
            x = ops.ln_star(x3_in, W[p + "feedforward.layernorm.gamma"], W[p + "feedforward.layernorm.beta"])
        logits = ops.lin(x, W[dec + "out.weight"], W[dec + "out.bias"], False)                 # every position; the loss keeps the non-zero targets
        lm, dlogits = ops.lm_nll(logits, tgt, keep_tok)
        zero = ops.zeros((1,))

        def backward(w_lm, w_att2=0.0, w_grd=0.0, w_cls=0.0):
            grads = {}
            dx = self._lin_bwd(ops.scale(dlogits, w_lm), x, W, dec + "out", grads)
            denc = {}
            for l in (1, 0):
                t = tape[l]
                p = t["p"]
                dx3_in, dg_, db_ = ops.ln_star_bwd(dx, t["x3_in"], W[p + "feedforward.layernorm.gamma"])
                self._acc(grads, p + "feedforward.layernorm.gamma", dg_)
                self._acc(grads, p + "feedforward.layernorm.beta", db_)
                df1 = ops.relu_bwd(self._lin_bwd(D_(dx3_in, "tfm", "tfm_res", l * 3 + 2), t["f1"], W, p + "feedforward.layer.linear2", grads), t["f1"])
                dx2 = ops.add(dx3_in, self._lin_bwd(df1, t["x2"], W, p + "feedforward.layer.linear1", grads))
                dx2_in, dg_, db_ = ops.ln_star_bwd(dx2, t["x2_in"], W[p + "attention.layernorm.gamma"])
                self._acc(grads, p + "attention.layernorm.gamma", dg_)
                self._acc(grads, p + "attention.layernorm.beta", db_)
                dc = self._lin_bwd(D_(dx2_in, "tfm", "tfm_res", l * 3 + 1), t["c"], W, p + "attention.layer.wo", grads)
                dq2, dk2, dv2 = ops.mha_bwd(dc, t["q2"], t["k2"], t["v2"], t["c"], t["lse2"], False, scale, p_att, seed, site(l, 1), it)
                dx1 = ops.add(dx2_in, self._lin_bwd(dq2, t["x1"], W, p + "attention.layer.wq", grads))
                de = ops.add(self._lin_bwd(dk2, t["e"], W, p + "attention.layer.wk", grads), self._lin_bwd(dv2, t["e"], W, p + "attention.layer.wv", grads))
                denc[enc[l]] = de if enc[l] not in denc else ops.add(denc[enc[l]], de)      # d enc = dK Wk + dV Wv, summed over the layers
                dx1_in, dg_, db_ = ops.ln_star_bwd(dx1, t["x1_in"], W[p + "selfattn.layernorm.gamma"])
                self._acc(grads, p + "selfattn.layernorm.gamma", dg_)
                self._acc(grads, p + "selfattn.layernorm.beta", db_)
                da = self._lin_bwd(D_(dx1_in, "tfm", "tfm_res", l * 3), t["a"], W, p + "selfattn.layer.wo", grads)
                dq, dk, dv = ops.mha_bwd(da, t["q"], t["k"], t["v"], t["a"], t["lse"], True, scale, p_att, seed, site(l, 0), it)
                dx = dx1_in
                for nm, g in (("wq", dq), ("wk", dk), ("wv", dv)):
                    dx = ops.add(dx, self._lin_bwd(g, t["x"], W, p + "selfattn.layer.%s" % nm, grads))
            demb = D_(dx, "tfm", "tfm_embed").reshape(B * L, H)
            self._acc(grads, dec + "out.weight", ops.scale(ops.index_add_rows(V, s_in, demb), math.sqrt(H)))     # the tied embedding
            self._prologue_bwd(pt, W, opt, grads, D_, dconv=denc.get("conv"), dpool_feats=denc.get("pool_feats"))
            return grads

        return [lm, zero, zero, zero], backward

    def forward_backward(self, W, opt, inp, n_replicas=1, host=None):
        """loss = (lm + w_att2 att2 + w_grd grd + w_cls cls) / n_replicas with the zero-weight terms dropped (main.py:238-255).
        opt.disable_caption (main.py:243-246): the language loss leaves the objective and the returned lm is 0; the logit head gets no
        gradient (absent from `grads`), the tensors only the language loss reached get exact zeros, as in the reference."""
        ops = self.ops
        caption = check_disable_caption(opt)
        losses, backward = self.forward(W, opt, inp, host)
        lm, att2_loss, grd_loss, cls_loss = losses
        loss = lm if caption else None
        for w, l in ((opt.w_att2, att2_loss), (opt.w_grd, grd_loss), (opt.w_cls, cls_loss)):
            if w:
                loss = ops.scale(l, w) if loss is None else ops.add(loss, ops.scale(l, w))
        loss = ops.scale(loss, 1.0 / n_replicas)
        c0 = 1.0 / n_replicas
        grads = backward(c0 if caption else 0.0, opt.w_att2 * c0, opt.w_grd * c0, opt.w_cls * c0)
        if not caption:
            losses = [ops.zeros((1,)), att2_loss, grd_loss, cls_loss]          # lm_loss.fill_(0), main.py:246
        return losses, loss, grads

    def step(self, W, opt, inp, lr=5e-4, betas=(0.9, 0.999), eps=1e-8, grad_clip=0.1, n_replicas=1, host=None, all_reduce=None):
        """forward_backward + (optional) gradient all-reduce + clip_grad_norm_ + first Adam step with one group per tensor and
        lr x0.1 for 'ctx2pool_grd' / 'vis_embed' (main.py:238-266,660-677).  `all_reduce(flat_tensor)` is the D1 hook: one
        sum-all-reduce of the flat fp32 gradient buffer (torch.distributed over NCCL in the product)."""
        ops = self.ops
        losses, loss, grads = self.forward_backward(W, opt, inp, n_replicas, host)
        keys = sorted(grads.keys())
        if all_reduce is not None:
            flat = ops.cat([grads[k].reshape(-1) for k in keys], 0)
            flat = all_reduce(flat)
            o = 0
            for k in keys:
                n = grads[k].numel()
                grads[k] = flat[o:o + n].reshape(tuple(grads[k].shape)).contiguous()
                o += n
        sq = None
        for k in keys:
            s = ops.sum_all(ops.mul(grads[k], grads[k]))
            sq = s if sq is None else ops.add(sq, s)
        total_norm = float(ops.to_host(sq)) ** 0.5
        coef = min(grad_clip / (total_norm + 1e-6), 1.0)
        new = {}
        for k in keys:
            step_lr = lr * 0.1 if ("ctx2pool_grd" in k or "vis_embed" in k) else lr
            new[k] = ops.adam_first_step(W[k], grads[k], coef, step_lr, betas[0], betas[1], eps)
        return losses, loss, grads, total_norm, new


class Trainer:
    """The reference's optimisation loop body (main.py:235-266 + the optimiser set-up of main.py:660-677) on flat device buffers.

    Every trainable tensor of the state_dict lives in ONE flat fp32 parameter buffer (`flat_w`, state_dict order); gradients, Adam's first
    and second moments are flat buffers with the same layout.  A step is

        forward (train mode) -> four losses -> explicit backward -> gradients into `flat_g`
        [world > 1]  ONE sum-all-reduce of `flat_g` (NCCL over NVLink; SURVEY.md 8e — the gradients were pre-divided by the replica
                     count like main.py:255, so the sum is nn.DataParallel's averaged gradient)
        gvd_tr_grad_norm  (global norm + clip coefficient, stays on the device)   -> clip_grad_norm_(grad_clip)   main.py:265
        gvd_tr_adam_flat  (torch.optim.Adam arithmetic, per-tensor lr table, step t) -> optimizer.step()          main.py:266
          (optim = 'sgd' / 'adamax': gvd_tr_sgd_flat / gvd_tr_adamax_flat, torch.optim.SGD(momentum=0.9) / Adamax, main.py:671-677)
        BatchNorm running statistics (train-mode side effect of model.py:114; rank-local like DataParallel's replica 0)

    `W` (the dict handed out by `.weights`) holds VIEWS into `flat_w`, so a module whose parameters are re-pointed at them
    (`adopt_module`) trains in place.  Tensors that receive no gradient keep lr 0 in the table and come out of a step unchanged, as
    torch.optim.Adam skips them: core.i2h_2 / h2h_2 (quirk Q10) from the start, and whatever else the last backward left out (with
    att_model = 'transformer': the top-down core, its embedding and heads, and the branch att_input_mode does not read; with
    opt.disable_caption: the logit head).

    optim: 'adam' (default), 'sgd' or 'adamax' — the three optimisers of main.py:671-677, with the same param groups, lr, weight_decay and betas
    (main.py:660-669; SGD ignores betas, as torch does).  The optimiser state lives in `flat_m` (Adam exp_avg, SGD momentum_buffer, Adamax
    exp_avg) and `flat_v` (Adam exp_avg_sq, Adamax exp_inf).  SGD and Adamax keep torch's per-tensor step count in `seg_step` (device int32,
    one entry per tensor), so a tensor's momentum buffer / bias correction starts with its own first gradient."""

    OPTIMS = ("adam", "sgd", "adamax")
    SGD_MOMENTUM = 0.9                                             # optim.SGD(params, momentum=0.9), main.py:673

    def __init__(self, ops, state_dict, opt, lr=5e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, grad_clip=0.1, all_reduce=None,
                 n_replicas=1, optim="adam"):
        if optim not in self.OPTIMS:
            raise ValueError("optim must be one of %s (main.py:671-677), got %r" % (", ".join(repr(o) for o in self.OPTIMS), optim))
        check_disable_caption(opt)
        self.optim = optim
        self.ops, self.opt = ops, opt
        self.step_fn = TrainStep(ops)
        self.lr, self.betas, self.eps, self.weight_decay, self.grad_clip = lr, betas, eps, weight_decay, grad_clip
        self.all_reduce, self.n_replicas = all_reduce, n_replicas
        self.t = 0
        self.keys = [k for k, v in state_dict.items() if torch.is_tensor(v) and v.is_floating_point() and "running_" not in k]
        self.never = ("core.i2h_2", "core.h2h_2")
        self.idle = frozenset()                                    # keys the last backward gave no gradient
        self._adopted = weakref.WeakSet()
        offs, o = {}, 0
        for k in self.keys:
            offs[k] = o
            o += (state_dict[k].numel() + 3) // 4 * 4             # 16-byte aligned segments (float4 loads in the norm kernel)
        self.offsets, self.numel = offs, o
        dev = ops.device
        self.flat_w = torch.zeros(o, dtype=torch.float32, device=dev)
        self.flat_g = torch.zeros(o, dtype=torch.float32, device=dev)
        self.flat_m = torch.zeros(o, dtype=torch.float32, device=dev)
        self.flat_v = torch.zeros(o, dtype=torch.float32, device=dev)
        self.norm = torch.zeros(2, dtype=torch.float32, device=dev)
        self.weights = {}
        for k in self.keys:
            n = state_dict[k].numel()
            view = self.flat_w[offs[k]:offs[k] + n].view(state_dict[k].shape)
            view.copy_(state_dict[k].detach().to(device=dev, dtype=torch.float32))
            self.weights[k] = view
        self.buffers = {k: state_dict[k].detach().clone().to(dev) for k in state_dict if k not in self.weights}
        ends = [offs[k] + (state_dict[k].numel() + 3) // 4 * 4 for k in self.keys]
        self.seg_end = torch.tensor(ends, dtype=torch.int64, device=dev)
        self.seg_step = torch.zeros(len(self.keys), dtype=torch.int32, device=dev)
        self.set_lr(lr)

    def set_lr(self, lr):
        """One param group per tensor; 'ctx2pool_grd' / 'vis_embed' fine-tune at lr x 0.1 (main.py:663-669); utils.set_lr decay = call again."""
        self.lr = lr
        lrs = [0.0 if (k in self.idle or k.startswith(self.never)) else (lr * 0.1 if ("ctx2pool_grd" in k or "vis_embed" in k) else lr) for k in self.keys]
        self.seg_lr = torch.tensor(lrs, dtype=torch.float32, device=self.ops.device)

    def grad_view(self, k):
        n = self.weights[k].numel()
        return self.flat_g[self.offsets[k]:self.offsets[k] + n].view(self.weights[k].shape)

    def adopt_module(self, module):
        """Re-point an nn.Module's parameters (and their .grad) at the flat buffers, and its buffers (BatchNorm running statistics) at this
        Trainer's: `loss.backward(); optimizer.step()` drivers and this Trainer then share storage, and the module decodes with the trained state."""
        for k, p in module.named_parameters():
            if k in self.weights:
                p.data = self.weights[k]
                p.grad = self.grad_view(k)
        for k, b in module.named_buffers():
            if k in self.buffers and self.buffers[k].shape == b.shape:
                b.data = self.buffers[k]
        self._adopted.add(module)

    def state_dict(self):
        sd = {k: v.detach().clone() for k, v in self.weights.items()}
        sd.update({k: v.detach().clone() for k, v in self.buffers.items()})
        return sd

    def forward_backward(self, inp, host=None):
        """Losses + gradients into flat_g (pre-divided by n_replicas, main.py:255); no optimiser step."""
        W = dict(self.weights)
        W.update(self.buffers)
        losses, loss, grads = self.step_fn.forward_backward(W, self.opt, inp, self.n_replicas, host)
        self.flat_g.zero_()
        for k, g in grads.items():
            self.grad_view(k).copy_(g.reshape(self.weights[k].shape))
        idle = frozenset(k for k in self.keys if k not in grads)
        if idle != self.idle:
            self.idle = idle
            self.set_lr(self.lr)
        return losses, loss

    def step(self, inp, host=None):
        """One optimisation step; returns (losses[4], loss).  The global gradient norm of the step is in `self.norm[0]` (device)."""
        losses, loss = self.forward_backward(inp, host)
        if self.all_reduce is not None:
            self.all_reduce(self.flat_g)                          # D1: ONE collective on the flat gradient buffer
        self.apply()
        return losses, loss

    def apply(self):
        """clip_grad_norm_ + the optimiser step on the flat buffers + the BatchNorm running statistics of the last forward."""
        ops = self.ops
        self.t += 1
        ops.grad_norm_(self.flat_g, self.grad_clip, self.norm)
        if self.optim == "adam":
            ops.adam_flat_(self.flat_w, self.flat_g, self.flat_m, self.flat_v, self.seg_end, self.seg_lr, self.norm, self.betas[0], self.betas[1],
                           self.eps, self.weight_decay, self.t)
        elif self.optim == "sgd":
            ops.sgd_flat_(self.flat_w, self.flat_g, self.flat_m, self.seg_end, self.seg_lr, self.seg_step, self.norm, self.SGD_MOMENTUM,
                          self.weight_decay)
        else:
            ops.adamax_flat_(self.flat_w, self.flat_g, self.flat_m, self.flat_v, self.seg_end, self.seg_lr, self.seg_step, self.norm, self.betas[0],
                             self.betas[1], self.eps, self.weight_decay)
        # the optimiser kernel writes the weights behind torch's back: bump the version counters of adopted modules' parameters, so that
        # code keyed on them (the module's cached native weights, AttModel._native_model) sees the new values
        for m in self._adopted:
            for k, p in m.named_parameters():
                if k in self.weights:
                    torch.autograd.graph.increment_version(p)
        if getattr(self.step_fn, "last_bn", None) is not None:
            mu, var, n = self.step_fn.last_bn
            rm, rv = self.buffers["att_embed_aux.0.running_mean"], self.buffers["att_embed_aux.0.running_var"]
            rm.copy_(ops.add(ops.scale(rm, 0.9), ops.scale(mu, 0.1)))
            rv.copy_(ops.add(ops.scale(rv, 0.9), ops.scale(var, 0.1 * n / (n - 1.0))))
            if "att_embed_aux.0.num_batches_tracked" in self.buffers:
                self.buffers["att_embed_aux.0.num_batches_tracked"] += 1
