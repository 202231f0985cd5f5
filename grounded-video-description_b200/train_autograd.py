"""`forward(..., 'MLE')` in train mode as ONE autograd node (SURVEY.md 8 row T7): the reference driver does

    lm, att2, grd, cls = model(..., 'MLE');  loss = (lm.sum() + w_att2*att2.sum() + ...) / lm.numel();  loss.backward()

(main.py:238-262).  `MLEFunction` keeps that contract on top of the explicit backward of gvd_b200.train: its forward returns the
four losses, its backward receives their four upstream gradients — the weights of the caller's combination — and runs the
hand-written backward ONCE with those weights (it is linear in them), handing every parameter its gradient.

A loss without `lm` (--disable_caption, main.py:243-246) reaches backward with g_lm = 0: the logit head's .grad stays None, and the tensors
only the language loss reached get exact-zero gradients rather than None, as in the reference, whose decode state torch.stack([h_att, h_lang])
(AttModel.py:163) carries a zero gradient into the language LSTM.

Verified on the CPU with the torch mock of the primitives (tests/test_train_host_logic.py) and on the device (tests/test_gpu_zz_train.py)."""
import torch


class MLEFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, step, opt, inp, host, keys, extra, *params):
        W = dict(zip(keys, params))
        W.update(extra or {})
        losses, backward = step.forward(W, opt, inp, host)
        ctx.backward_fn, ctx.keys, ctx.shapes = backward, keys, [tuple(p.shape) for p in params]
        return tuple(l.reshape(1).clone() for l in losses)

    @staticmethod
    def backward(ctx, g_lm, g_att2, g_grd, g_cls):
        w = [0.0 if g is None else float(g.reshape(-1)[0]) for g in (g_lm, g_att2, g_grd, g_cls)]
        grads = ctx.backward_fn(*w)
        out = []
        for k, shp in zip(ctx.keys, ctx.shapes):
            g = grads.get(k)
            out.append(None if g is None else g.reshape(shp))
        return (None, None, None, None, None, None) + tuple(out)


def mle_losses(step, opt, inp, host, named_params, extra=None):
    """named_params: iterable of (key, tensor); tensors that do not require grad are passed through unchanged.  extra: non-parameter
    state_dict entries (buffers) the forward may read."""
    keys = [k for k, _ in named_params]
    params = [p for _, p in named_params]
    return MLEFunction.apply(step, opt, inp, host, keys, extra, *params)


def update_bn_running_stats(step, running_mean, running_var, momentum=0.1):
    """nn.BatchNorm1d train-mode side effect (model.py:114): running = (1 - m) running + m batch, the variance unbiased."""
    ops = step.ops
    mu, var, n = step.last_bn
    running_mean.copy_(ops.add(ops.scale(running_mean, 1.0 - momentum), ops.scale(mu, momentum)))
    running_var.copy_(ops.add(ops.scale(running_var, 1.0 - momentum), ops.scale(var, momentum * n / (n - 1.0))))
