"""float64 restatement of lifting's device arithmetic (csrc/lift.cu, include/xunet_b200.h "Lifting"): the camera and timestep
draw, the noise, the guided and weighted residual with its image gradient, and the render backward of a given image gradient
(autograd through tests/field_ref.py).  The GPU tests compare the kernels against it; the CPU tests check it against
synthetic._look_at, finite differences and closed forms."""
import math

import numpy as np
import torch

from tests import field_ref as F
from tests import pose_ref as PR
from tests.device_data_ref import mix64

M64 = (1 << 64) - 1
SEED_DOMAIN = 0x6C6966745F736473
MAX_RESIDUAL = 16.0
U1, U2 = 0x5851F42D4C957F2D, 0x14057B7EF767814F


def draw_hash(seed: int, i: int, p: int) -> int:
    return PR.draw_hash((seed ^ SEED_DOMAIN) & M64, i, p)


def uniform(h: int, k: int) -> float:
    return (mix64((h + k) & M64) >> 11) * 2.0 ** -53


def band_basis(up):
    """(up, e1, e2): up normalised, e1 the first basis vector of least |up_j| made perpendicular to up, e2 = up x e1."""
    up = np.asarray(up, np.float64)
    up = up / math.sqrt(float(up @ up))
    j = int(np.argmin(np.abs(up)))
    e1 = np.eye(3)[j] - up[j] * up
    e1 = e1 / math.sqrt(float(e1 @ e1))
    return up, e1, np.cross(up, e1)


def look_at(c, up, e1):
    """[right down f] (columns) of the camera at c looking at the origin with world up `up`; when f is (nearly) parallel to
    up, right is e1 made perpendicular to f."""
    c = np.asarray(c, np.float64)
    f = -c / math.sqrt(float(c @ c))
    right = np.cross(f, up)
    rn = math.sqrt(float(right @ right))
    if rn < 1e-6:
        right = e1 - float(e1 @ f) * f
        rn = math.sqrt(float(right @ right))
    right = right / rn
    return np.stack([right, np.cross(f, right), f], axis=1)


def draw(seed: int, i: int, P: int, t_min: int, t_max: int, up, elev_deg, radius: float):
    """(t (P,), R (P,3,3), c (P,3)) of iteration i (1-based), in fp64."""
    up, e1, e2 = band_basis(up)
    s_lo, s_hi = math.sin(math.radians(elev_deg[0])), math.sin(math.radians(elev_deg[1]))
    ts, Rs, cs = [], [], []
    for p in range(P):
        h = draw_hash(seed, i, p)
        ts.append(t_min + h % (t_max - t_min + 1))
        s = s_lo + (s_hi - s_lo) * uniform(h, U1)
        phi = 2.0 * math.pi * uniform(h, U2)
        c = radius * (s * up + math.sqrt(max(0.0, 1.0 - s * s)) * (math.cos(phi) * e1 + math.sin(phi) * e2))
        Rs.append(look_at(c, up, e1))
        cs.append(c)
    return np.array(ts, np.int64), np.stack(Rs), np.stack(cs)


def noise(render, t, seed: int, i: int, sqrt_ac, sqrt_1mac):
    """(eps (P,S,S,3), z (P,S,S,3), logsnr (P,)) of the P drawn renders (P,S,S,3) in [-1, 1]."""
    render = np.asarray(render, np.float64)
    P = len(t)
    eps = np.stack([PR.hash_normal(draw_hash(seed, i, p), render[p].size).reshape(render[p].shape) for p in range(P)])
    sa = np.asarray(sqrt_ac, np.float64)[t].reshape(P, 1, 1, 1)
    sb = np.asarray(sqrt_1mac, np.float64)[t].reshape(P, 1, 1, 1)
    return eps, sa * render + sb * eps, PR.logsnr(t)


def eps_hat(out_c, out_u, z, t, w: float, prediction: str, sqrt_ac, sqrt_1mac):
    """The guided output (1 + w) o_c - w o_u read as eps: as is, or sqrt(1 - abar) z + sqrt(abar) o_g for prediction='v'."""
    og = (1.0 + w) * np.asarray(out_c, np.float64) - w * np.asarray(out_u, np.float64)
    if prediction == 'eps':
        return og
    P = len(t)
    sa = np.asarray(sqrt_ac, np.float64)[t].reshape(P, 1, 1, 1)
    sb = np.asarray(sqrt_1mac, np.float64)[t].reshape(P, 1, 1, 1)
    return sb * np.asarray(z, np.float64) + sa * og


def grad_unit(sds_weight: float, recon_weight: float) -> float:
    """The smallest power of two u with (32 sds_weight + 2 recon_weight) / u <= 2^23 (1 when both weights are 0)."""
    l1 = 2.0 * MAX_RESIDUAL * sds_weight + 2.0 * recon_weight
    return 1.0 if l1 == 0.0 else 2.0 ** math.ceil(math.log2(l1 / 2.0 ** 23))


def image_grad(out, z, eps, render, x, t, w: float, prediction: str, sds_weight: float, recon_weight: float, sqrt_ac, sqrt_1mac):
    """(dC (P+1,S,S,3), sds, recon): dC_p = 2 sds_weight omega_t r / (3 S^2 P) with r = clamp(eps_hat - eps) and omega_t =
    sqrt_1mac[t]^2, dC_P = 2 recon_weight (C - u) / (3 S^2) for the source view; sds = mean r^2, recon = mean (C - u)^2.  dC
    is the gradient itself: the kernel writes dC / unit."""
    P = len(t)
    out = np.asarray(out, np.float64)
    S = out.shape[1]
    r = eps_hat(out[:P], out[P:], z, t, w, prediction, sqrt_ac, sqrt_1mac) - np.asarray(eps, np.float64)
    r = np.clip(np.where(np.isfinite(r), r, 0.0), -MAX_RESIDUAL, MAX_RESIDUAL)
    omega = (np.asarray(sqrt_1mac, np.float64)[t] ** 2).reshape(P, 1, 1, 1)
    C = (np.asarray(render, np.float64)[P] + 1.0) / 2.0
    d = C - np.clip((np.asarray(x, np.float64) + 1.0) / 2.0, 0.0, 1.0)
    dC = np.concatenate([2.0 * sds_weight * omega * r / (3 * S * S * P), (2.0 * recon_weight * d / (3 * S * S))[None]])
    return dC, float(np.mean(r ** 2)), float(np.mean(d ** 2))


def render_backward(grid, dC, R, t, K, bound, near, step, background, tv=(0.0, 0.0), unit=1.0):
    """d/d(grid) [unit sum dC . C + TV]: the gradient xunet_field_image_grad writes, by autograd through field_ref's renderer.
    Non-finite values of dC (V,S,S,3) are read as 0, as the kernel does."""
    g = torch.as_tensor(grid, dtype=torch.float64).detach().requires_grad_(True)
    dC = torch.as_tensor(np.asarray(dC), dtype=torch.float64)
    dC = unit * torch.where(torch.isfinite(dC), dC, torch.zeros_like(dC))
    S = dC.shape[1]
    pix = F.render(g, R, t, K, S, bound, near, step, background)
    C = (pix + 1) / 2
    (grad,) = torch.autograd.grad((C * dC).sum() + F.tv(g, *tv), g)
    return grad


def samples_per_word(R, t, K, S, G, bound, near, step):
    """(G, G, G) int: the number of samples of all V S S rays that fall in the (up to 8) cells around each grid point, i.e. how
    many fixed-point roundings each word of the backward's scatter receives (each sample's contribution is rounded on its
    own).  Computed in fp64; the kernel's fp32 sample positions can move a sample across a cell face, so callers double it."""
    o, d = F.rays(R, t, K, S)
    o, d = o.reshape(-1, 3), d.reshape(-1, 3)
    t0, L, hit = F.segments(o, d, bound, near)
    n = torch.where(hit, torch.clamp(torch.ceil(L / step), min=1), torch.zeros_like(L)).long()
    counts = torch.zeros((G - 1) ** 3, dtype=torch.int64)
    for r in torch.nonzero(hit).flatten().tolist():
        k = torch.arange(int(n[r]), dtype=torch.float64)
        dk = torch.where(k < n[r] - 1, torch.full_like(k, step), L[r] - (n[r] - 1) * step)
        tm = t0[r] + k * step + 0.5 * dk
        u = ((o[r] + tm[:, None] * d[r] + bound) * ((G - 1) / (2 * bound))).clamp(0, G - 1)
        i0 = torch.clamp(torch.floor(u), max=G - 2).long()
        counts += torch.bincount((i0[:, 0] * (G - 1) + i0[:, 1]) * (G - 1) + i0[:, 2], minlength=(G - 1) ** 3)
    c = torch.nn.functional.pad(counts.reshape(G - 1, G - 1, G - 1), (1, 1, 1, 1, 1, 1))
    w = sum(c[a:a + G, b:b + G, e:e + G] for a in (0, 1) for b in (0, 1) for e in (0, 1))
    return w
