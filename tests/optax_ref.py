"""CPU restatements of the optax pieces behind gradient clipping and learning-rate warm-up, next to the oracle's
`adam_update` (oracle/xunet_ref.py): what the clip / warm-up tests hold the CUDA path to.  optax is not installable here, so
these are restated from its published sources."""
import math


def clip_by_global_norm(grads, max_norm):
    """optax.clip_by_global_norm(max_norm) on a dict (or list) of gradient leaves: g_norm = sqrt(sum of all squares);
    the leaves are returned unchanged if g_norm < max_norm, else as (g / g_norm) * max_norm.  Returns (clipped, g_norm).
    The norm is summed in float64 here (optax sums in the leaves' dtype, in XLA's order)."""
    leaves = grads.values() if isinstance(grads, dict) else grads
    g_norm = math.sqrt(math.fsum(float((g.double() ** 2).sum()) for g in leaves))
    if g_norm < max_norm:
        return grads, g_norm
    f = lambda g: (g / g_norm) * max_norm
    return ({k: f(g) for k, g in grads.items()} if isinstance(grads, dict) else [f(g) for g in grads]), g_norm


def warmup_lr(lr, count, warmup_steps):
    """optax.linear_schedule(0, lr, warmup_steps) at the schedule's count (0 for the first update): lr * min(count, W) / W,
    and the constant lr when W == 0.  optax evaluates it as (0 - lr) * (1 - count / W) + lr, equal up to rounding."""
    if warmup_steps == 0:
        return lr
    return lr * min(count, warmup_steps) / warmup_steps
