"""``AttModel`` — the reference's nn.Module surface (misc/model.py:28-742) over the native hot path.

What is kept from the reference: the constructor signature and the ``opt`` fields it reads
(model.py:29-73), the parameter tree / state_dict keys (checkpoint contract, main.py:638), the
``forward(segs_feat, seq, gt_seq, num, ppls, gt_boxes, mask_boxes, ppls_feat, frm_mask,
sample_idx, pnt_mask, opt, eval_opt={})`` dispatch on 'MLE' | 'GRD' | 'sample' (model.py:227-234)
and the return tuples.  What is new: all arithmetic runs in hand-written sm_90a kernels behind
the C-ABI (include/gvd_b200.h); the three copies of the prologue (model.py:302-409, 504-568,
634-698) are one native call; nothing executes on the CPU and there is no torch fallback.
"""
import math
import os
import pickle
import warnings

import torch
import torch.nn as nn

try:                                   # imported as gvd_b200.misc.model
    from .. import capi
    from .CaptionModelBU import CaptionModel
    from .transformer import Transformer, TransformerDecoder
except ImportError:                    # imported as top-level ``misc.model`` (drop-in layout)
    import capi
    from misc.CaptionModelBU import CaptionModel
    from misc.transformer import Transformer, TransformerDecoder


def _seq(*mods):
    return nn.Sequential(*mods)


def check_sample_n(n):
    """eval_opt['sample_n'] as an int >= 1 (captions sampled per clip); ValueError for anything else (bool, float, < 1)."""
    if isinstance(n, bool) or not hasattr(n, "__index__"):
        raise ValueError("sample_n must be an integer >= 1 (got %r)" % (n,))
    n = int(n.__index__())
    if n < 1:
        raise ValueError("sample_n must be an integer >= 1 (got %r)" % (n,))
    return n


class AttModel(CaptionModel):
    def __init__(self, opt):
        super().__init__()
        self.vocab_size = opt.vocab_size
        self.detect_size = opt.detect_size
        self.input_encoding_size = opt.input_encoding_size
        self.rnn_size = opt.rnn_size
        self.num_layers = opt.num_layers
        self.drop_prob_lm = opt.drop_prob_lm
        self.seq_length = opt.seq_length
        self.seg_info_size = 50
        self.fc_feat_size = opt.fc_feat_size + self.seg_info_size
        self.att_feat_size = opt.att_feat_size
        self.att_hid_size = opt.att_hid_size
        self.seq_per_img = opt.seq_per_img
        self.itod = opt.itod
        self.att_input_mode = opt.att_input_mode
        self.region_attn_mode = getattr(opt, "region_attn_mode", "mix")
        self.transfer_mode = opt.transfer_mode
        self.test_mode = opt.test_mode
        self.enable_BUTD = opt.enable_BUTD
        self.w_grd = opt.w_grd
        self.w_cls = opt.w_cls
        self.num_sampled_frm = opt.num_sampled_frm
        self.num_prop_per_frm = opt.num_prop_per_frm
        self.att_model = opt.att_model
        self.unk_idx = int(opt.wtoi["UNK"])
        self.t_attn_size = opt.t_attn_size
        self.min_value = -1e8
        opt.beta = 1                      # side effect of the reference constructor (model.py:72)
        self.beta = 1
        self._dims = capi.dims_from_opt(opt)      # raises NotImplementedError for modes off the hot path
        import types
        self.opt_ns = types.SimpleNamespace(rnn_size=opt.rnn_size, seq_length=opt.seq_length, vocab_size=opt.vocab_size,
                                            num_sampled_frm=opt.num_sampled_frm, obj_interact=getattr(opt, "obj_interact", False),
                                            att_input_mode=self.att_input_mode, region_attn_mode=self.region_attn_mode)
        self.vis_encoding_size = 2048
        # BUTD: the region features are fc7 alone (model.py:65-69); the reference asserts att_input_mode 'region' (dims_from_opt)
        self.pool_feat_size = self.att_feat_size if self.enable_BUTD else self.att_feat_size + 300 + self.detect_size + 1

        H, A, E = self.rnn_size, self.att_hid_size, self.input_encoding_size
        p = self.drop_prob_lm
        # parameter tree: same module nesting as the reference => same state_dict keys
        self.loc_fc = _seq(nn.Linear(5, 300), nn.ReLU(), nn.Dropout())
        self.embed = _seq(nn.Embedding(self.vocab_size, E), nn.ReLU(), nn.Dropout(p))
        self.vis_embed = _seq(nn.Embedding(self.detect_size + 1, self.vis_encoding_size), nn.ReLU(), nn.Dropout(p))
        self.fc_embed = _seq(nn.Linear(self.fc_feat_size, H), nn.ReLU(), nn.Dropout(p))
        self.seg_info_embed = _seq(nn.Linear(4, self.seg_info_size), nn.ReLU(), nn.Dropout(p))
        self.att_embed = nn.ModuleList([_seq(nn.Linear(2048, H // 2), nn.ReLU(), nn.Dropout(p)),
                                        _seq(nn.Linear(opt.fc_feat_size - 2048, H // 2), nn.ReLU(), nn.Dropout(p))])
        self.att_embed_aux = _seq(nn.BatchNorm1d(H), nn.ReLU())
        self.pool_embed = _seq(nn.Linear(self.pool_feat_size, H), nn.ReLU(), nn.Dropout(p))
        self.ctx2att = nn.Linear(H, A)
        self.ctx2pool = nn.Linear(H, A)
        self.logit = nn.Linear(H, self.vocab_size)
        if opt.obj_interact:
            self.obj_interact = Transformer(H, 0, 0, d_hidden=int(H / 2), n_layers=2, n_heads=6, drop_ratio=0.2, pe=False)
        if self.att_model == "transformer":          # language decoder (model.py:137-143); runs through csrc/gvd_tfm.cu
            self.cap_model = TransformerDecoder(H, 0, self.vocab_size, d_hidden=H // 2, n_layers=2, n_heads=6, drop_ratio=0.2)
        self.context_enc = nn.GRU(H, H // 2, 2, dropout=0.2, bidirectional=True, batch_first=True)
        self.ctx2pool_grd = _seq(nn.Linear(self.att_feat_size, self.vis_encoding_size), nn.ReLU(), nn.Dropout(p))
        if self.transfer_mode == "cls":             # transfer_mode 'none' builds no class bias (model.py:180-215)
            self.vis_classifiers_bias = nn.Parameter(torch.zeros(self.detect_size + 1))
        self._init_from_detectron(opt)

        self._native = None
        self._native_sig = None
        self._tfm = None

    # ------------------------------------------------------------------ constructor side effects
    def _init_from_detectron(self, opt):
        """fc7 / class-score transfer from ``data/detectron_weights/*.pkl`` (CWD-relative, as in the
        reference: model.py:173-211).  Missing files only warn: checkpoints overwrite these values.
        transfer_mode 'none' transfers fc7 only: vis_embed keeps its default init (model.py:214-215)."""
        d = "data/detectron_weights"
        try:
            names = ("fc7_w", "fc7_b") + (("cls_score_w", "cls_score_b") if self.transfer_mode == "cls" else ())
            w = {k: pickle.load(open(os.path.join(d, k + ".pkl"), "rb")) for k in names}
        except (FileNotFoundError, OSError):
            warnings.warn("data/detectron_weights/*.pkl not found: ctx2pool_grd / vis_embed keep their default init "
                          "(load a checkpoint before use)")
            return
        with torch.no_grad():
            fs = self.att_feat_size
            self.ctx2pool_grd[0].weight[:fs].copy_(torch.from_numpy(w["fc7_w"]))
            self.ctx2pool_grd[0].bias[:fs].copy_(torch.from_numpy(w["fc7_b"]))
            if self.transfer_mode != "cls":
                return
            cw, cb = torch.from_numpy(w["cls_score_w"]), torch.from_numpy(w["cls_score_b"])
            assert len(opt.itod) + 1 == opt.glove_clss.size(0)
            assert len(opt.vg_cls) == opt.glove_vg_cls.size(0)
            vg = opt.glove_vg_cls / opt.glove_vg_cls.norm(dim=1, keepdim=True)
            ours = opt.glove_clss / opt.glove_clss.norm(dim=1, keepdim=True)
            self.max_sim, self.matched_cls = (vg @ ours.t()).max(dim=0)     # nearest VG class per target class
            idx = self.matched_cls.clone()
            idx[0] = 0                                                     # background row
            self.vis_embed[0].weight.copy_(cw[idx])
            self.vis_classifiers_bias.copy_(cb[idx])

    # ------------------------------------------------------------------ native plumbing
    def _native_model(self):
        """(Re)upload weights when any parameter tensor changed (version counters / storage)."""
        dev_params = list(self.state_dict(keep_vars=True).items())
        if not all(t.is_cuda for _, t in dev_params):
            raise capi.GvdError("model parameters are not on a CUDA device: call model.cuda() "
                                "(gvd_b200 has no CPU path)")
        sig = tuple((t.data_ptr(), t._version) for _, t in dev_params)
        if self._native is None:
            self._native = capi.NativeModel(self._opt_view())
        if sig != self._native_sig:
            self._native.load_state_dict({k: t for k, t in dev_params})
            if self.att_model == "transformer":
                if self._tfm is None:
                    self._tfm = capi.TransformerCaptioner(self.rnn_size, self.vocab_size, self.seq_length, n_heads=6)
                self._tfm.load_state_dict({k: t for k, t in dev_params})
            self._native_sig = sig
        return self._native

    def _opt_view(self):
        class _O:
            pass
        o = _O()
        d = self._dims
        o.vocab_size, o.detect_size, o.input_encoding_size = d.vocab_size, d.detect_size, d.input_encoding_size
        o.rnn_size, o.att_hid_size, o.seq_length = d.rnn_size, d.att_hid_size, d.seq_length
        o.num_sampled_frm, o.num_prop_per_frm = d.num_sampled_frm, d.num_prop_per_frm
        o.att_feat_size, o.fc_feat_size, o.obj_interact = d.att_feat_size, d.fc_feat_size, bool(d.obj_interact)
        o.wtoi = {"UNK": str(d.unk_idx)}
        o.att_model, o.att_input_mode = self.att_model, self.att_input_mode     # the language LSTM's input (AttModel.py:144-156)
        o.region_attn_mode = self.region_attn_mode                              # the region attention's score (AttModel.py:79-96)
        o.transfer_mode = self.transfer_mode                                    # whether the similarity has a class bias (model.py:84-85)
        o.enable_BUTD = self.enable_BUTD                                        # fc7-only region features (model.py:65-69)
        return o

    @staticmethod
    def _u8(mask):
        return mask if mask.dtype == torch.uint8 else mask.to(torch.uint8)

    # ------------------------------------------------------------------ the reference's entry point
    def forward(self, segs_feat, seq, gt_seq, num, ppls, gt_boxes, mask_boxes, ppls_feat, frm_mask, sample_idx, pnt_mask, opt,
                eval_opt={}):
        """eval_opt['video_idx'] (int64 [B]): a video-indexed batch of B events.  segs_feat then holds the frame features of V videos
        [V,T,F], passed once per video, and event b is the window sample_idx[b] of video video_idx[b]; every other tensor is per event.
        The result equals the same call on segs_feat[video_idx] without the key.  Top-down captioner in eval mode only."""
        video_idx = eval_opt.get("video_idx") if eval_opt else None
        if video_idx is not None:
            if self.att_model == "transformer":
                raise NotImplementedError("video_idx: the transformer captioner's cross-attention reads per-clip frame encodings; pass "
                                          "segs_feat[video_idx] without the key")
            if self.training:
                raise NotImplementedError("video_idx is an inference batch layout; training batches are random events: pass "
                                          "segs_feat[video_idx] without the key")
            if not torch.is_tensor(video_idx) or video_idx.device != segs_feat.device:
                raise ValueError("video_idx must be a tensor on the device of segs_feat (%s)" % segs_feat.device)
        if opt == "MLE":
            return self._forward(segs_feat, seq, gt_seq, ppls, gt_boxes, mask_boxes, num, ppls_feat, frm_mask, sample_idx, pnt_mask,
                                 video_idx=video_idx)
        elif opt == "GRD":
            return self._forward(segs_feat, seq, gt_seq, ppls, gt_boxes, mask_boxes, num, ppls_feat, frm_mask, sample_idx, pnt_mask, True,
                                 video_idx=video_idx)
        elif opt == "sample":
            if self.att_model == "transformer":
                # the reference cannot return here: it unpacks four values from the three its _sample returns in this mode (model.py:233,578);
                # repaired contract = _sample's triple (seq [B,L], zeros [B,1], zeros [B,1])
                return self._sample(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, eval_opt)
            seq, seqLogprobs, att2, sim_mat = self._sample(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, eval_opt)
            return seq, att2, sim_mat
        raise ValueError("unknown forward mode %r (expected 'MLE', 'GRD' or 'sample')" % (opt,))

    def _prologue(self, segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, beam=1, nbox=0, video_idx=None, att2=False, rows=1):
        nm = self._native_model()
        sim = nm.prologue(segs_feat.float().contiguous(), ppls.float().contiguous(), num.long().contiguous(),
                          ppls_feat.float().contiguous(), sample_idx.long().contiguous(), self._u8(pnt_mask).contiguous(),
                          want_sim=not self.enable_BUTD,       # BUTD (transformer only): nothing reads the similarity, so it is not computed
                          beam=beam, nbox=nbox, att2=att2, rows=rows,   # the workspace is sized for the decode that follows
                          video_idx=video_idx.contiguous() if video_idx is not None else None)
        return nm, sim

    def _sample(self, segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, opt={}):
        """Beam search, greedy or multinomial decode (model.py:492-624, 627-742), dispatched in the reference's order: beam_size > 1 ->
        beam search whatever sample_max is (model.py:501); the transformer captioner decodes greedily whatever sample_max is
        (model.py:570-578); sample_max = 1 -> greedy; sample_max = 0 -> multinomial sampling at eval_opt['temperature'] (model.py:595-603).

        Sampling draws from softmax(logits / temperature) like the reference's torch.multinomial, but through counter-based noise keyed by
        a per-call seed (gvd_decode_sample): the seed is one draw from torch's default CPU generator, so torch.manual_seed(s) reproduces a
        call and successive calls differ.  The draws of a row depend on its index in the batch: splitting a batch changes them.

        eval_opt['att2_weights'] = True asks for the region-attention logits [B,L,R] of the returned captions as the second output of
        'sample', the input of extract_grounding.  Greedy and multinomial decoding return them anyway; beam search then returns them
        instead of its region index per word (see _sample_beam).

        eval_opt['sample_n'] = n (sample_max = 0): n sampled captions per clip from one prologue.  seq, the log-probs and the att2 logits then
        have B * n rows, caption j of clip b in row b * n + j; sim_mat stays [B, D+1, R], once per clip.  The draws equal the same call on
        the batch repeated with repeat_interleave(n, 0) under the same seed (gvd_decode_sample_n), and with video_idx the rows are events x n.
        extract_grounding then takes ppls.repeat_interleave(n, 0).  n = 1 (or no key) is the plain call; n > 1 is refused with sample_max = 1
        (n identical greedy captions) and with beam_size > 1 (ValueError), and by the transformer captioner (NotImplementedError), which
        decodes greedily whatever sample_max is."""
        sample_max = opt.get("sample_max", 1)
        beam_size = opt.get("beam_size", 1)
        temperature = opt.get("temperature", 1.0)
        video_idx = opt.get("video_idx")
        sample_n = check_sample_n(opt.get("sample_n", 1))
        if sample_n > 1:
            if beam_size > 1:
                raise ValueError("sample_n > 1 draws several sampled captions per clip; beam search (beam_size=%r) returns one" % (beam_size,))
            if self.att_model == "transformer":
                raise NotImplementedError("sample_n: the transformer captioner decodes greedily whatever sample_max is (model.py:570-578)")
            if sample_max:
                raise ValueError("sample_n > 1 needs sample_max = 0: greedy decoding would give %d identical captions per clip" % sample_n)
        if opt.get("att2_weights") and self.att_model == "transformer":
            raise NotImplementedError("att2_weights: the transformer captioner has no region attention to return (its 'sample' returns zeros "
                                      "there, model.py:578)")
        if beam_size > 1:
            if self.att_model == "transformer":
                raise NotImplementedError("the transformer captioner decodes greedily (Decoder.greedy, transformer.py:214); the reference has no "
                                          "beam search for it either (model.py:627-742 is top-down only)")
            return self._sample_beam(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, opt)
        if self.training:
            raise capi.GvdError("'sample' runs in eval mode (main.py:315); call model.eval()")
        B, T = ppls.size(0), segs_feat.size(1)
        if self.att_model == "transformer":
            nm, _ = self._prologue(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask)
            seq = self._tfm.decode_greedy(*self._tfm_encodings(nm, B, T))
            zero = seq.new_zeros(B, 1)
            return seq, zero, zero.clone()                # model.py:578
        if not sample_max:
            temperature = float(temperature)
            if not (math.isfinite(temperature) and temperature > 0):
                raise ValueError("temperature must be finite and > 0 (got %r)" % (temperature,))
            seed = int(torch.randint(0, 2 ** 62, (1,)))
        nm, sim = self._prologue(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, video_idx=video_idx, rows=sample_n)
        mask = self._u8(pnt_mask).contiguous()
        if sample_max:
            seq, logp, att2 = nm.decode_greedy(B, T, mask)
        elif sample_n > 1:
            seq, logp, att2 = nm.decode_sample_n(B, T, sample_n, mask, seed, temperature)
        else:
            seq, logp, att2 = nm.decode_sample(B, T, mask, seed, temperature)
        return seq, logp, att2, sim

    def _tfm_encodings(self, nm, B, T):
        """The encoder outputs of the two decoder layers (model.py:571-576): views into the prologue's workspace."""
        conv = lambda: nm.workspace_tensor(B, T, "conv_feats", (B, T, self.rnn_size))
        pool = lambda: nm.workspace_tensor(B, T, "pool_feats", (B, nm.R, self.rnn_size))
        if self.att_input_mode == "both":
            return conv(), pool()
        if self.att_input_mode == "featmap":
            c = conv()
            return c, c
        p = pool()
        return p, p

    def extract_grounding(self, att2_weights, input_ppls):
        """main.py:364-370 on the device (SURVEY.md 8(f) rank 2): for every generated word and sampled frame the proposal with
        the largest region-attention logit.  att2_weights [B,L,R] (second output of 'sample'), input_ppls [B,R,7]
        -> (att2_ind [B,L,F] int64, obj_bbox_att2 [B,L,F,7]), the two tensors the reference driver builds with
        torch.max / permute / gather before its per-word Python loop."""
        F, P = int(self.num_sampled_frm), int(self.num_prop_per_frm)
        return capi.grounding_extract(att2_weights.float().contiguous(), input_ppls.float().contiguous(), F, P)

    def _sample_beam(self, segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, opt={}):
        """Beam search (model.py:627-742 + CaptionModelBU.py:24-185), all clips batched on the device.

        The reference crashes here as shipped (12 arguments into the 10-argument core, and `forward`
        unpacks 4 values from the 3 returned); this implements the documented minimal repair
        (SURVEY.md App. A.5 / B D1-D4) and returns 4 values so that `forward(..., 'sample')` works:
        (seq, seqLogprobs, att2 region INDEX per word [B,L], sim_mat).

        opt['att2_weights'] = True: the third value is instead the region-attention logits [B,L,R] fp32 of each returned caption, the
        grounding that greedy decoding returns: row t is the masked logit row the caption's own beam used to pick word t (row 0 the <bos>
        step, later rows those of the beam's ancestors, found through the search's parent pointers), rows after the caption's last word 0.
        They equal the logits of the teacher-forced pass on the caption, and feed extract_grounding as they are."""
        beam_size = opt.get("beam_size", 10)
        att2 = bool(opt.get("att2_weights", False))
        if self.training:
            raise capi.GvdError("'sample' runs in eval mode (main.py:315); call model.eval()")
        B, T = ppls.size(0), segs_feat.size(1)
        nm, sim = self._prologue(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, beam=beam_size, video_idx=opt.get("video_idx"), att2=att2)
        mask = self._u8(pnt_mask).contiguous()
        if att2:
            seq, logp, _, att2_w = nm.beam_decode_att2(B, T, beam_size, mask)
            return seq, logp, att2_w, sim
        seq, logp, att = nm.beam_decode(B, T, beam_size, mask)
        return seq, logp, att, sim

    def _forward_train(self, segs_feat, input_seq, gt_seq, ppls, gt_boxes, mask_boxes, num, ppls_feat, frm_mask, sample_idx, pnt_mask):
        """Train-mode 'MLE' (model.py:283-483 with BatchNorm batch statistics and train-mode Dropout): the four losses as ONE autograd node
        whose backward is the explicit device backward (gvd_b200/train.py), so the reference driver's
        `loss.backward(); clip_grad_norm_; optimizer.step()` (main.py:238-266) works unchanged.

        Dropout: the reference's masks come from torch's global RNG; here they are counter-based Philox masks keyed by
        (`self.dropout_seed`, site, step) at the same sites with the same probabilities (drop_prob_lm, 0.5 for loc_fc, 0.2 inside
        obj_interact and between the GRU layers).  `self.train_dropout = False` switches every site off — the deterministic mode in
        which losses and gradients are pinned to the reference."""
        try:                               # imported as gvd_b200.misc.model
            from ..train import TrainStep
            from ..train_autograd import mle_losses, update_bn_running_stats
            from ..train_ops import NativeOps
        except ImportError:                # top-level ``misc.model`` (drop-in layout: the package directory is on sys.path)
            from train import TrainStep
            from train_autograd import mle_losses, update_bn_running_stats
            from train_ops import NativeOps
        if getattr(self, "_train_step", None) is None:
            self._train_step = TrainStep(NativeOps())
        if getattr(self, "train_dropout", True):
            seed = getattr(self, "dropout_seed", None)
            if seed is None:
                seed = self.dropout_seed = int(torch.initial_seed()) & 0x7FFFFFFFFFFFFFFF
            self._train_step.dropout = dict(seed=seed, p_lm=float(self.drop_prob_lm), p_interact=0.2, p_gru=0.2, p_loc=0.5)
        else:
            self._train_step.dropout = None
        V, D = self.vocab_size, self.detect_size
        f32 = lambda t: t.float().contiguous()
        inp = dict(segs_feat=f32(segs_feat), ppls=f32(ppls), num=num.long().contiguous(), ppls_feat=f32(ppls_feat),
                   sample_idx=sample_idx.long().contiguous(), pnt_mask=self._u8(pnt_mask).contiguous(), gt_seq=gt_seq.long().contiguous(),
                   input_seq=input_seq.long().contiguous(), frm_mask=self._u8(frm_mask).contiguous(), gt_boxes=f32(gt_boxes),
                   mask_boxes=self._u8(mask_boxes).contiguous())
        host = dict(gt_seq=inp["gt_seq"].cpu(), input_seq=inp["input_seq"].cpu(), sample_idx=inp["sample_idx"].cpu())    # drive the control flow
        self._check_ids(host["gt_seq"][:, 0], host["input_seq"][:, 0, :, 0])
        named = [(k, p) for k, p in self.named_parameters()]
        W_extra = {k: v for k, v in self.state_dict(keep_vars=True).items() if "running_" in k}
        losses = mle_losses(self._train_step, self.opt_ns, inp, host, named, W_extra)
        if self.att_input_mode != "dual_region":        # dual_region never runs att_embed_aux (model.py:393): its statistics stay
            with torch.no_grad():
                update_bn_running_stats(self._train_step, self.att_embed_aux[0].running_mean, self.att_embed_aux[0].running_var)
                self.att_embed_aux[0].num_batches_tracked += 1
        return losses

    def _forward_tfm(self, segs_feat, gt_seq, ppls, num, ppls_feat, sample_idx, pnt_mask):
        """att_model='transformer' branch of _forward (model.py:411-419): the teacher-forced language loss and five zeros ("Masked Transformer
        does not support box supervision yet"); 'GRD' takes the same branch in the reference.  Eval-mode arithmetic (no dropout).  The training
        step of this captioner is gvd_b200.train.Trainer (TrainStep's transformer branch); train mode through this module is refused."""
        if self.training:
            raise NotImplementedError("the transformer captioner trains through gvd_b200.train.Trainer (adopt_module(model) shares the weights "
                                      "with this module), not through model.train() + 'MLE'; call model.eval() for the teacher-forced loss")
        B, T = segs_feat.size(0), segs_feat.size(1)
        seq = torch.cat((gt_seq.new_zeros(B, 1), gt_seq[:, 0, :]), dim=1).long().contiguous()          # model.py:285-286
        if seq.numel() and (int(seq.min()) < 0 or int(seq.max()) >= self.vocab_size):
            raise IndexError("caption token id outside [0, %d)" % self.vocab_size)
        nm, _ = self._prologue(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask)
        lm = self._tfm.teacher_loss(*self._tfm_encodings(nm, B, T), seq.to(segs_feat.device))
        z = lambda: lm.new_zeros(1)
        return lm, z(), z(), z(), z(), z()

    def _check_ids(self, words, input_cls):
        """nn.Embedding raises IndexError on out-of-range ids (model.py:79,93); the native gathers must never see them."""
        V, D = self.vocab_size, self.detect_size
        if words.numel() and (int(words.min()) < 0 or int(words.max()) >= V):
            raise IndexError("caption token id outside [0, %d)" % V)
        if input_cls.numel() and (int(input_cls.min()) < 0 or int(input_cls.max()) > V + D):
            raise IndexError("input_seq word/class id outside [0, %d]" % (V + D))

    def _forward(self, segs_feat, input_seq, gt_seq, ppls, gt_boxes, mask_boxes, num, ppls_feat, frm_mask, sample_idx, pnt_mask,
                 eval_obj_ground=False, video_idx=None):
        """Teacher-forced pass (model.py:283-489): 'MLE' -> (lm, att2, ground, cls) losses each of shape (1,)
        (model.py:483); 'GRD' -> (cls_pred [N,2] or 0 in test_mode, att2 idx [B,S,10], grounding idx [B,S,10]).
        model.eval(): eval-mode arithmetic through gvd_teacher_fwd; model.train() + 'MLE': the training forward with its explicit backward
        (`_forward_train`); 'GRD' is an evaluation mode (main.py:90,125)."""
        if self.att_model == "transformer":
            return self._forward_tfm(segs_feat, gt_seq, ppls, num, ppls_feat, sample_idx, pnt_mask)
        if self.training:
            if eval_obj_ground:
                raise capi.GvdError("'GRD' runs in eval mode (main.py:90); call model.eval()")
            return self._forward_train(segs_feat, input_seq, gt_seq, ppls, gt_boxes, mask_boxes, num, ppls_feat, frm_mask, sample_idx, pnt_mask)
        B, T, L = ppls.size(0), segs_feat.size(1), self.seq_length
        seq = torch.cat((gt_seq.new_zeros(B, 1), gt_seq[:, 0, :]), dim=1).long().contiguous()          # model.py:285-286
        col_any = (seq[:, 1:L] != 0).any(dim=0)                                                          # model.py:425 early exit
        dead = (~col_any).nonzero()
        S = int(dead[0]) + 1 if dead.numel() else L
        input_cls = input_seq[:, 0, :, 0].long().contiguous()
        self._check_ids(seq, input_cls)
        nbox = gt_boxes.size(1)
        pm = self._u8(pnt_mask).contiguous()
        nm, _ = self._prologue(segs_feat, ppls, num, ppls_feat, sample_idx, pnt_mask, nbox=nbox, video_idx=video_idx)
        fmask = self._u8(frm_mask).contiguous()
        if not eval_obj_ground:
            mb = self._u8(mask_boxes)[:, 0].contiguous()                                                 # seq_per_img == 1
            losses = nm.teacher_forward(B, T, S, 0, seq, input_cls, ppls.float().contiguous(), gt_boxes.float().contiguous(), mb, fmask, pm)
            return losses[0:1], losses[1:2], losses[2:3], losses[3:4]
        att_idx, grd_idx, sim_target, pred = nm.teacher_forward(B, T, S, 1, seq, input_cls, ppls.float().contiguous(),
                                                                gt_boxes.float().contiguous(), None, fmask, pm)
        if self.test_mode:
            cls_pred = 0
        else:
            pos = sim_target > 0                                                                        # model.py:346,353-355
            cls_pred = torch.stack((sim_target[pos].long(), pred.unsqueeze(1).expand_as(sim_target)[pos].long()), dim=1)
        return cls_pred, att_idx, grd_idx
