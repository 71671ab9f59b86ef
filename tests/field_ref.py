"""float64 torch restatement of the radiance grid of xunet_field_render / xunet_field_loss_grad (include/xunet_b200.h states
the definition), differentiable w.r.t. the grid by autograd."""
import math

import torch
import torch.nn.functional as F

DENSITY_SHIFT = -6.0
MIN_GRID, MAX_GRID = 2, 256
MAX_BOUND = 64.0
MAX_SAMPLES = 4096
MAX_RAYS = 1 << 20
FIXED_ONE = 2.0 ** 32


def rays(R, t, K, S):
    """Origins and directions (V, S, S, 3) of every pixel: t_v and normalize(R_v K_v^-1 (col + 1/2, row + 1/2, 1))."""
    R, t, K = (torch.as_tensor(x, dtype=torch.float64) for x in (R, t, K))
    row, col = torch.meshgrid(torch.arange(S, dtype=torch.float64) + 0.5, torch.arange(S, dtype=torch.float64) + 0.5,
                              indexing='ij')
    p = torch.stack([col, row, torch.ones_like(row)], -1)
    d = torch.einsum('vij,vjk,hwk->vhwi', R, torch.linalg.inv(K), p)
    d = d / torch.linalg.norm(d, dim=-1, keepdim=True)
    return t[:, None, None, :].expand_as(d), d


def segments(o, d, bound, near):
    """(t0, L, hit) of rays (M, 3): the part of the ray inside [-b, b]^3 at t >= near."""
    lo = torch.full(o.shape[:1], float(near), dtype=torch.float64)
    hi = torch.full(o.shape[:1], math.inf, dtype=torch.float64)
    ok = torch.ones(o.shape[:1], dtype=torch.bool)
    for a in range(3):
        da, oa = d[:, a], o[:, a]
        zero = da == 0
        sd = torch.where(zero, torch.ones_like(da), da)
        t1, t2 = (-bound - oa) / sd, (bound - oa) / sd
        lo = torch.where(zero, lo, torch.maximum(lo, torch.minimum(t1, t2)))
        hi = torch.where(zero, hi, torch.minimum(hi, torch.maximum(t1, t2)))
        ok &= ~(zero & (oa.abs() > bound))
    hit = ok & (hi > lo)
    return lo, torch.where(hit, hi - lo, torch.zeros_like(lo)), hit


def composite(grid, o, d, bound, near, step, background, chunk=4096):
    """C (M, 3) in [0, 1] of rays o, d (M, 3) through grid (G, G, G, 4)."""
    out = [_composite(grid, o[i:i + chunk], d[i:i + chunk], bound, near, step, background) for i in range(0, len(o), chunk)]
    return torch.cat(out) if out else torch.zeros(0, 3, dtype=torch.float64)


def _composite(grid, o, d, bound, near, step, background):
    G = grid.shape[0]
    t0, L, hit = segments(o, d, bound, near)
    n = torch.where(hit, torch.clamp(torch.ceil(L / step), min=1), torch.zeros_like(L)).long()
    nmax = max(int(n.max()) if len(n) else 0, 1)
    k = torch.arange(nmax, dtype=torch.float64)[None]
    nf = n.to(torch.float64)[:, None]
    valid = k < nf
    dk = torch.where(k < nf - 1, torch.full_like(k, step), L[:, None] - (nf - 1) * step)
    dk = torch.where(valid, dk, torch.zeros_like(dk))
    tm = t0[:, None] + k * step + 0.5 * dk
    u = ((o[:, None, :] + tm[..., None] * d[:, None, :] + bound) * ((G - 1) / (2 * bound))).clamp(0, G - 1)
    i0 = torch.clamp(torch.floor(u), max=G - 2).long()
    f = u - i0
    flat = grid.reshape(-1, 4)
    raw = 0
    for c in range(8):
        bits = [(c >> 2) & 1, (c >> 1) & 1, c & 1]
        w = 1
        idx = 0
        for a in range(3):
            w = w * (f[..., a] if bits[a] else 1 - f[..., a])
            idx = idx * G + (i0[..., a] + bits[a])
        raw = raw + w[..., None] * flat[idx]
    sigma = F.softplus(raw[..., 0] + DENSITY_SHIFT)
    col = torch.sigmoid(raw[..., 1:])
    a = -torch.expm1(-sigma * dk)
    a = torch.where(valid, a, torch.zeros_like(a))
    trans = torch.cumprod(torch.cat([torch.ones_like(a[:, :1]), 1 - a], 1), 1)      # T_0 .. T_n
    C = (trans[:, :-1, None] * a[..., None] * col).sum(1)
    return C + trans[:, -1:] * (background + 1) / 2


def render(grid, R, t, K, S, bound, near, step, background):
    """(V, S, S, 3) in [-1, 1]."""
    o, d = rays(R, t, K, S)
    C = composite(grid, o.reshape(-1, 3), d.reshape(-1, 3), bound, near, step, background)
    return (2 * C - 1).reshape(o.shape)


def tv(grid, tv_density, tv_color):
    G = grid.shape[0]
    s = 0
    for a in range(3):
        dlt = torch.diff(grid, dim=a) ** 2
        s = s + tv_density * dlt[..., 0].sum() + tv_color * dlt[..., 1:].sum()
    return s / G ** 3


def data_loss(grid, views, R, t, K, pixels, bound, near, step, background):
    """(1/3N) sum (C - u)^2 over the training pixels `pixels` (indices v S S + row S + col) of views (V, S, S, 3)."""
    views = torch.as_tensor(views, dtype=torch.float64)
    S = views.shape[1]
    o, d = rays(R, t, K, S)
    pixels = torch.as_tensor(pixels, dtype=torch.long)
    C = composite(grid, o.reshape(-1, 3)[pixels], d.reshape(-1, 3)[pixels], bound, near, step, background)
    u = ((views.reshape(-1, 3)[pixels] + 1) / 2).clamp(0, 1)
    return ((C - u) ** 2).sum() / (3 * len(pixels))
