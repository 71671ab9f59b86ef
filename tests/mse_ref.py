"""Reference of the mean-squared epsilon loss next to the oracle's Frobenius loss (oracle/xunet_ref.py loss_fn): the value,
and every parameter gradient through torch autograd on the oracle's forward."""
from collections import OrderedDict

import torch

from oracle import xunet_ref as R


def mse_loss(eps_hat, noise, w=None):
    """L = (1/B) sum_b w_b * mean_i (eps_hat - noise)_bi^2 (w = None: all 1): DDPM's L_simple, weighted per sample."""
    r = (eps_hat - noise).reshape(eps_hat.shape[0], -1)
    per_sample = (r * r).mean(dim=1)
    if w is not None:
        per_sample = per_sample * torch.as_tensor(w, dtype=per_sample.dtype)
    return per_sample.mean()


def loss_and_grads(params, batch, noise, cond_mask, cfg: R.RefConfig = R.SMALL, *, loss='frobenius', loss_weight=None,
                   train=True, drop_mask_fn=None):
    """R.loss_and_grads with the choice of loss: 'frobenius' (the oracle's own) or 'mse' (mse_loss with loss_weight).
    Returns (loss, flat grads dict, eps_hat)."""
    if loss == 'frobenius':
        assert loss_weight is None
        return R.loss_and_grads(params, batch, noise, cond_mask, cfg, train=train, drop_mask_fn=drop_mask_fn)
    assert loss == 'mse', loss
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in R.flatten(params).items())
    eps_hat = R.xunet_forward(R.nest(leaves), batch, cond_mask, cfg, train=train, drop_mask_fn=drop_mask_fn)
    value = mse_loss(eps_hat, noise.to(eps_hat.dtype), loss_weight)
    grads = torch.autograd.grad(value, list(leaves.values()), allow_unused=True)
    gd = OrderedDict((k, torch.zeros_like(v) if g is None else g) for (k, v), g in zip(leaves.items(), grads))
    return value.detach(), gd, eps_hat.detach()
