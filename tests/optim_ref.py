"""The two flat optimiser primitives of the SGD / Adamax training loop (main.py:671-677) as torch definitions — TEST INFRASTRUCTURE.

`OptimRefOps` is the CPU mock `TorchRefOps` plus `sgd_flat_` / `adamax_flat_`: tests/test_optim_host_logic.py runs gvd_b200.train.Trainer with it
against torch.optim, and tests/test_gpu_optim.py checks the native kernels (csrc/gvd_train.cu) against the same functions."""
import torch

from ops_ref import TorchRefOps


def _per_elem(w, seg_end, seg_lr, seg_step):
    """Per-element learning rate and step count (the steps taken before this one) of the flat segment layout."""
    lr, steps = torch.zeros_like(w), torch.zeros(w.numel(), dtype=torch.int64, device=w.device)
    lo = 0
    for e, l, s in zip(seg_end.tolist(), seg_lr.tolist(), seg_step.tolist()):
        lr[lo:e], steps[lo:e] = l, s
        lo = e
    return lr, steps


class OptimRefOps(TorchRefOps):
    def sgd_flat_(self, w, g, buf, seg_end, seg_lr, seg_step, norm, momentum, weight_decay):
        """torch.optim.SGD(momentum, dampening=0, nesterov=False) on flat buffers with a per-segment lr and step count; lr <= 0 = idle."""
        if norm is not None:
            g.mul_(norm[1])
        lr, steps = _per_elem(w, seg_end, seg_lr, seg_step)
        live = lr > 0
        d = g + weight_decay * w if weight_decay else g
        b = torch.where(steps == 0, d, momentum * buf + d)                 # torch creates the buffer on the tensor's first step
        buf.copy_(torch.where(live, b, buf))
        w.sub_(torch.where(live, lr * buf, torch.zeros_like(w)))
        seg_step += (seg_lr > 0).to(seg_step.dtype)

    def adamax_flat_(self, w, g, m, u, seg_end, seg_lr, seg_step, norm, b1, b2, eps, weight_decay):
        """torch.optim.Adamax on flat buffers with a per-segment lr and step count (bias correction per tensor); lr <= 0 = idle."""
        if norm is not None:
            g.mul_(norm[1])
        lr, steps = _per_elem(w, seg_end, seg_lr, seg_step)
        live = lr > 0
        d = g + weight_decay * w if weight_decay else g
        m.copy_(torch.where(live, b1 * m + (1 - b1) * d, m))
        u.copy_(torch.where(live, torch.maximum(b2 * u, d.abs() + eps), u))
        clr = (lr.double() / (1 - b1 ** (steps + 1).double())).float()
        w.sub_(torch.where(live, clr * (m / u), torch.zeros_like(w)))
        seg_step += (seg_lr > 0).to(seg_step.dtype)
