"""Reference vector-Jacobian product of the X-UNet forward (what xunet_backward_vjp computes): torch autograd on the oracle's
xunet_forward, seeded with a given d_eps = dL/d(eps_hat), giving dL/dparams and dL/dx, dL/dz of the two input views."""
from collections import OrderedDict

import torch

from oracle import xunet_ref as R


class InputSTE(R.Bf16Emulation):
    """Bf16Emulation, except that the packed input views (B,2,S,S,3) are rounded like a _RoundSTE operand: the value is rounded
    to bf16, the gradient passes through unrounded.  That is the engine's contract for dx / dz in bf16 mode (they come straight
    from fp32 accumulators); the oracle's own policy stores the input tensor with _Store, whose backward rounds."""

    def __init__(self, x, z):
        self._stack = torch.stack([x.detach(), z.detach()], dim=1)

    def store(self, t):
        if t.shape == self._stack.shape and torch.equal(t.detach(), self._stack.to(t.dtype)):
            return R._RoundSTE.apply(t)
        return R._Store.apply(t)


def vjp(params, batch, cond_mask, d_eps, cfg: R.RefConfig, *, train=False, drop_mask_fn=None, bf16_inputs_ste=False):
    """Returns (eps_hat, OrderedDict of parameter gradients, dx, dz) of L = <d_eps, eps_hat>.  The parameters and the batch are
    used in their own dtype (fp64 for the reference); bf16_inputs_ste=True evaluates the rounding-aware forward (InputSTE)."""
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in R.flatten(params).items())
    x = batch['x'].detach().clone().requires_grad_(True)
    z = batch['z'].detach().clone().requires_grad_(True)
    emu = InputSTE(x, z) if bf16_inputs_ste else None
    eps = R.xunet_forward(R.nest(leaves), dict(batch, x=x, z=z), cond_mask, cfg, train=train, drop_mask_fn=drop_mask_fn, emu=emu)
    value = (eps * d_eps.to(eps.dtype)).sum()
    grads = torch.autograd.grad(value, list(leaves.values()) + [x, z], allow_unused=True)
    gp = OrderedDict((k, torch.zeros_like(v) if g is None else g) for (k, v), g in zip(leaves.items(), grads))
    return eps.detach(), gp, grads[-2], grads[-1]
