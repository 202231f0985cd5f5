"""Specification of the transformer captioner's training step and the torch mock of its attention primitive — TEST INFRASTRUCTURE.

`tfm_train_step` is the counterpart of the oracle's `train_step` for att_model = 'transformer': the train-mode prologue, the teacher-forced
decoder of TransformerDecoder.forward (misc/transformer.py:207-212,276-283) with a `drop` hook at its three Dropout sites, loss = lm / n_replicas
(model.py:411-419 returns the language loss alone), autograd, clip_grad_norm_ and the first Adam step with one group per tensor
(main.py:660-677).  tests/golden/make_golden_tfm_train.py pins it to the unmodified reference; tests/test_tfm_train_host_logic.py checks it and
the product's orchestration against each other.

`TfmRefOps` adds `mha_fwd` / `mha_bwd` (the definition of gvd_tr_mha_fwd / _bwd) to the primitive mock of tests/ops_ref.py."""
import math

import torch
import torch.nn.functional as F

import gvd_oracle as O
from ops_ref import TorchRefOps


def _id_drop(x, kind, site, sub=0):
    return x


def tfm_decoder(W, enc, s_in, drop=None):
    """Decoder.forward (transformer.py:207-212) over the input tokens s_in [B, S]: embedding with the tied out.weight * sqrt(d_model) plus the
    positional encoding, then 2 DecoderLayers (causal self-attention `dots - triu(1) * 1e10`, attention over enc[l], feed-forward), each
    sub-block a ResidualBlock with the custom LayerNorm.  Dropout sites (p = 0.2, model.py:137-142), through `drop(x, 'tfm', site, sub)`:
    tfm_embed (:209), tfm_attn on each head's probabilities (:105, sub = (layer * 2 + {0 self, 1 cross}) * 8 + head) and tfm_res in every
    ResidualBlock (:88, sub = layer * 3 + block).  Returns the last hidden state [B, S, H]."""
    drop = drop or _id_drop
    B, S = s_in.shape
    H = enc[0].shape[-1]
    sizes = O.head_chunks(H)
    scale = math.sqrt(H)
    Wout = W["cap_model.decoder.out.weight"]
    x = drop((Wout * math.sqrt(H))[s_in] + O.positional_encodings(S, H, s_in.device), "tfm", "tfm_embed")
    tri = torch.ones(S, S, device=s_in.device).triu(1) * 1e10

    def mh(p, qx, kx, l, cross):
        q, k, v = qx @ W[p + "wq.weight"].t(), kx @ W[p + "wk.weight"].t(), kx @ W[p + "wv.weight"].t()
        outs, o = [], 0
        for hi, sz in enumerate(sizes):
            dots = q[..., o:o + sz] @ k[..., o:o + sz].transpose(1, 2)
            if not cross:
                dots = dots - tri
            att = drop(torch.softmax(dots / scale, dim=-1), "tfm", "tfm_attn", (l * 2 + cross) * 8 + hi)
            outs.append(att @ v[..., o:o + sz])
            o += sz
        return torch.cat(outs, -1) @ W[p + "wo.weight"].t()

    for l in range(2):
        p = "cap_model.decoder.layers.%d." % l
        x = O._ln_star(x + drop(mh(p + "selfattn.layer.", x, x, l, 0), "tfm", "tfm_res", l * 3),
                       W[p + "selfattn.layernorm.gamma"], W[p + "selfattn.layernorm.beta"])
        x = O._ln_star(x + drop(mh(p + "attention.layer.", x, enc[l], l, 1), "tfm", "tfm_res", l * 3 + 1),
                       W[p + "attention.layernorm.gamma"], W[p + "attention.layernorm.beta"])
        f = O._lin(O._lin(x, W, p + "feedforward.layer.linear1", relu=True), W, p + "feedforward.layer.linear2")
        x = O._ln_star(x + drop(f, "tfm", "tfm_res", l * 3 + 2), W[p + "feedforward.layernorm.gamma"], W[p + "feedforward.layernorm.beta"])
    return x


def tfm_lm(W, opt, inp, feats, drop=None):
    """The language loss of model.py:411-419: cross-entropy over the positions whose target seq[:, 1:] is non-zero (mask(), transformer.py:51-54)."""
    enc = O.tfm_encodings(opt, feats)
    gt = inp["gt_seq"][:, :opt.seq_per_img, :].reshape(-1, inp["gt_seq"].shape[2])
    seq = torch.cat((torch.zeros(gt.shape[0], 1, dtype=gt.dtype, device=gt.device), gt), 1)
    s_in, tgt = seq[:, :-1], seq[:, 1:]
    x = tfm_decoder(W, enc, s_in, drop)
    keep = tgt != 0
    logits = x[keep] @ W["cap_model.decoder.out.weight"].t() + W["cap_model.decoder.out.bias"]
    return F.cross_entropy(logits, tgt[keep])


def tfm_train_step(W, opt, inp, lr=5e-4, betas=(0.9, 0.999), eps=1e-8, grad_clip=0.1, n_replicas=1, drop=None):
    """One optimisation step of the transformer captioner (main.py:235-266 with the four-loss unpacking the reference's driver cannot do for
    this branch): prologue with BatchNorm batch statistics, teacher-forced decoder, loss = lm / n_replicas, autograd (tensors the loss does
    not reach get no gradient), clip_grad_norm_(grad_clip), first Adam step.  Returns (lm, loss, grads{key}, total norm, new params{key})."""
    P = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running_" not in k else v) for k, v in W.items()}
    feats = O.prologue(P, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"], train_bn=True,
                       drop=drop)
    lm = tfm_lm(P, opt, inp, feats, drop)
    loss = lm / n_replicas
    keys = [k for k, v in P.items() if torch.is_tensor(v) and v.requires_grad]
    gl = torch.autograd.grad(loss, [P[k] for k in keys], allow_unused=True)
    grads = {k: g for k, g in zip(keys, gl) if g is not None}
    total_norm = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
    coef = torch.clamp(grad_clip / (total_norm + 1e-6), max=1.0)
    new = {}
    for k, g in grads.items():
        g = g * coef
        step_lr = lr * 0.1 if ("ctx2pool_grd" in k or "vis_embed" in k) else lr
        m = (1 - betas[0]) * g
        v = (1 - betas[1]) * g * g
        new[k] = W[k] - (step_lr / (1 - betas[0])) * m / (v.sqrt() / math.sqrt(1 - betas[1]) + eps)
    return lm.detach(), loss.detach(), grads, total_norm, new


class TfmRefOps(TorchRefOps):
    """TorchRefOps plus the decoder attention: a plain composition per torch.chunk head, with gvd_tr_dropout's mask on each head's
    contiguous [B, Lq, N] probabilities at site site_base + head."""

    def _heads(self, H):
        o = 0
        for s in O.head_chunks(H):
            yield o, s
            o += s

    def _probs(self, q, k, causal, scale, o, s):
        dots = (q[..., o:o + s] @ k[..., o:o + s].transpose(1, 2)) * scale
        if causal:
            Lq, N = dots.shape[1], dots.shape[2]
            dots = dots.masked_fill(torch.arange(N).view(1, N) > torch.arange(Lq).view(Lq, 1), float("-inf"))
        return dots

    def mha_fwd(self, q, k, v, causal, scale, p=0.0, seed=0, site_base=0, step=0):
        outs, lses = [], []
        for h, (o, s) in enumerate(self._heads(q.shape[-1])):
            dots = self._probs(q, k, causal, scale, o, s)
            a = torch.softmax(dots, dim=-1)
            if p > 0:
                a = self.dropout(a.contiguous(), p, seed, site_base + h, step)
            outs.append(a @ v[..., o:o + s])
            lses.append(torch.logsumexp(dots, dim=-1))
        return torch.cat(outs, -1), torch.stack(lses, 1)

    def mha_bwd(self, do, q, k, v, o_, lse, causal, scale, p=0.0, seed=0, site_base=0, step=0):
        dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
        for h, (o, s) in enumerate(self._heads(q.shape[-1])):
            a = torch.exp(self._probs(q, k, causal, scale, o, s) - lse[:, h].unsqueeze(-1))
            doh = do[..., o:o + s]
            ad, dad = a, doh @ v[..., o:o + s].transpose(1, 2)
            if p > 0:
                ad = self.dropout(a.contiguous(), p, seed, site_base + h, step)
                dad = self.dropout(dad.contiguous(), p, seed, site_base + h, step)
            dv[..., o:o + s] = ad.transpose(1, 2) @ doh
            ds = a * (dad - (a * dad).sum(-1, keepdim=True))
            dq[..., o:o + s] = (ds @ k[..., o:o + s]) * scale
            dk[..., o:o + s] = (ds.transpose(1, 2) @ q[..., o:o + s]) * scale
        return dq, dk, dv
