"""Regularisers / losses of the hot path with the reference's names (loss_functions/losses.py, train.py).

* ``grad_penalty_loss`` -- R1 (losses.py:87-99).  The double backward it needs is provided by construction: every op's
  backward in gif_b200.ops is itself built from differentiable ops.
* ``PathLengthRegularizor`` -- the reference's class (losses.py:102-124) is unrunnable against its own generator and
  would have a zero gradient if it ran (SURVEY 8 L2).  This implements the documented rule the survey adopted
  (PARITY UNPINNED): differentiate w.r.t. w = z_to_w(embd[idx]), keep the reference's noise normaliser
  (1/sqrt(numel(img)), batch included), batch-mean length, the EMA line as written, create_graph=True.
"""
import numpy as np
import torch
import torch.nn.functional as F
from torch.autograd import grad


def l2_reg(model):
    """losses.py:16-20."""
    reg = 0
    for param in model.parameters():
        reg = reg + torch.norm(param)
    return reg


def grad_penalty_loss(inputs, outs, step):
    """losses.py:87-99: per-sample weight * ||d sum(outs) / d input||^2 (weight 5.0 when step is None)."""
    from . import ops
    grad_penalty = 0
    for inp_idx, inpt in enumerate(inputs):
        with ops.input_gradient_only():          # d scores / d image: no convolution weight gradients on the way
            grad_real = grad(outputs=outs.sum(), inputs=inpt, create_graph=True)[0]
        if step is not None:
            w = 1 + step - inp_idx
            w = 0.05 / (w * np.log2(1 + w))
        else:
            w = 5.0
        grad_penalty = grad_penalty + w * (grad_real.reshape(grad_real.size(0), -1).norm(2, dim=1) ** 2)
    return grad_penalty


class PathLengthRegularizor:
    def __init__(self):
        self.pl_moving_mean = 0
        self.pl_decay = 0.01

    def path_length_reg(self, generator, step, alpha, input_indices, cond=None, pl_noise=None):
        """``generator``: a StyledGenerator (or a wrapper exposing ``.module``) in rendered-condition mode;
        ``cond``: its (B,6,H,W) condition.  Returns the scalar penalty (train.py:205-208 weights it by 2)."""
        g = generator.module if hasattr(generator, "module") else generator
        w = g.z_to_w(g.img_embdng(input_indices))
        fake = _synth_from_w(g, w, cond, step)
        return self.path_length_from(fake, w, pl_noise)

    def path_length_from(self, fake, w, pl_noise=None):
        """The penalty for images ``fake`` already synthesised (with a graph) from the latent ``w``."""
        if pl_noise is None:
            pl_noise = torch.randn(fake.shape, device=fake.device)
        pl_noise = pl_noise / np.sqrt(np.prod(fake.shape))                       # losses.py:114
        from . import ops
        with ops.input_gradient_only():          # d image / d w: the generator's weight gradients are not part of it
            pl_grads = grad(outputs=torch.sum(fake * pl_noise), inputs=w, create_graph=True)[0]
        pl_lengths = torch.mean(torch.sqrt(torch.sum(torch.pow(pl_grads, 2), dim=1)))   # losses.py:116
        # losses.py:119 as written (no stop-gradient: the new mean == decay * length and carries its gradient into the
        # penalty); only the value kept for the next call is detached so that no graph outlives the iteration.
        # The running mean lives in ONE persistent 0-d device tensor updated in place: a captured CUDA graph reads and
        # writes it at a fixed address (rebinding the attribute to a fresh tensor every call would leave a replayed
        # graph reading the freed tensor of capture time).
        if not torch.is_tensor(self.pl_moving_mean):
            self.pl_moving_mean = torch.full((), float(self.pl_moving_mean), dtype=pl_lengths.dtype, device=pl_lengths.device)
        ema = self.pl_moving_mean + self.pl_decay * pl_lengths - self.pl_moving_mean
        penalty = torch.pow(pl_lengths - ema, 2)                                 # losses.py:122
        self.pl_moving_mean.copy_(ema.detach())
        return penalty


def _synth_from_w(g, w, cond, step):
    """Runs the synthesis network of a StyledGenerator from a given w (B,512) with the condition pyramid."""
    from . import ops
    c = ops.to_nhwc(cond)
    noise = [ops.to_nchw_view(ops.cond_resize(c, 4 * 2 ** i)) for i in range(step + 1)]
    return g.generator([w], None, noise, step, 1)[0]


def d_logistic_loss(real_scores, fake_scores):
    """train.py:144,171-172."""
    return F.softplus(-real_scores).mean() + F.softplus(fake_scores).mean()


def g_nonsaturating_loss(fake_scores):
    """train.py:203."""
    return F.softplus(-fake_scores).mean()
