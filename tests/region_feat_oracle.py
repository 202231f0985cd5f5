"""The CPU oracle (oracle/gvd_oracle.py) for transfer_mode 'none' and enable_BUTD (model.py:65-69,84-85,180-215,357-364, opts.py:62,66).

'none' builds the module without vis_classifiers_bias.  The reference then computes the region-class similarity (model.py:326-336,524-533,
652-661) and the teacher-forced grounding logits (model.py:472-476) without the class bias; everything else is that of 'cls'.
The oracle reads W["vis_classifiers_bias"] at those two places.  ``oracle_weights(opt, W)`` adds it for 'none' as an integer zero vector:
adding it changes no float (x + 0 == x), and autograd gives an integer tensor no gradient, so ``O.train_step`` / ``tfm_train_step`` over
these weights is the training reference of 'none' (the bias takes no part in the gradient norm or the update).  For 'cls' it returns W.

enable_BUTD (with the transformer captioner's att_input_mode 'region'): the region features are pool_embed(fc7) alone, with no loc_fc, label
features or LayerNorms.  ``oracle_region_feats()`` puts that region embedding in place of the oracle's for the duration of a call; every
loop of the oracle (and tests/tfm_train_ref.py) reaches it through ``O.prologue``.  The similarity is still computed there but feeds nothing,
so autograd gives vis_embed and the class bias no gradient, as in the reference."""
import contextlib

import torch

import gvd_oracle as O


def oracle_weights(opt, W):
    if getattr(opt, "transfer_mode", "cls") != "none":
        return W
    assert "vis_classifiers_bias" not in W
    return dict(W, vis_classifiers_bias=torch.zeros(opt.detect_size + 1, dtype=torch.int64))


def _region_embedding(W, opt, ppls, g_pool, sim, drop=None):
    if not getattr(opt, "enable_BUTD", False):
        return _orig(W, opt, ppls, g_pool, sim, drop)
    drop = drop or O._id_drop
    return drop(O._lin(g_pool, W, "pool_embed.0", relu=True), "lm", "pool_embed")     # model.py:384 on fc7 alone


_orig = O.region_embedding


@contextlib.contextmanager
def oracle_region_feats():
    O.region_embedding = _region_embedding
    try:
        yield O
    finally:
        O.region_embedding = _orig
