"""float64 restatement of pose estimation's device arithmetic (csrc/pose_fit.cu, include/xunet_b200.h "Pose estimation"): the
draws, the loss and its seed, the tangent projection, the Adam step of xunet_adam_step and the retraction on SO(3).  The
GPU tests compare the kernels against it; the CPU tests check it against autograd, finite differences and scipy."""
import math

import numpy as np

from tests.device_data_ref import mix64
from tests.util import _mix64

M64 = (1 << 64) - 1
SMALL_ANGLE2 = 1e-6


def draw_hash(seed: int, i: int, p: int) -> int:
    return mix64((seed * 0x9E3779B97F4A7C15 + i * 0xD1B54A32D192ED03 + p) & M64)


def timesteps(seed: int, i: int, P: int, t_min: int, t_max: int, strata: int = 0) -> np.ndarray:
    """t_p of the P draws of iteration i (1-based): uniform from the hash, or stratified over `strata` draws."""
    span = t_max - t_min + 1
    if strata > 0:
        return np.array([t_min + (2 * (((i - 1) * P + p) % strata) + 1) * span // (2 * strata) for p in range(P)], np.int64)
    return np.array([t_min + draw_hash(seed, i, p) % span for p in range(P)], np.int64)


def hash_normal(seed: int, n: int) -> np.ndarray:
    """xu_hash_normal(seed, k) for k < n: Box-Muller on the same two 24-bit uniforms, in fp64 (the device rounds to fp32)."""
    k = np.arange(n, dtype=np.uint64)
    with np.errstate(over='ignore'):
        h1 = _mix64(np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(2) * k + np.uint64(1))
        h2 = _mix64(h1 + np.uint64(0xD1B54A32D192ED03))
    u1 = ((h1 >> np.uint64(40)).astype(np.float64) + 1.0) / 16777216.0
    u2 = (h2 >> np.uint64(40)).astype(np.float64) / 16777216.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * math.pi * u2)


def logsnr(t) -> np.ndarray:
    b = math.atan(math.exp(-10.0))
    a = math.atan(math.exp(10.0)) - b
    return -2.0 * np.log(np.tan(a * (np.asarray(t, np.float64) / 1000.0) + b))


def draw(y, H: int, P: int, seed: int, i: int, t_min: int, t_max: int, sqrt_ac, sqrt_1mac, prediction='eps', strata=0):
    """(t (P,), eps (P,S,S,3), z (H P,S,S,3), logsnr (H P,), target (P,S,S,3)) of iteration i, in fp64."""
    y = np.asarray(y, np.float64)
    t = timesteps(seed, i, P, t_min, t_max, strata)
    eps = np.stack([hash_normal(draw_hash(seed, i, p), y.size).reshape(y.shape) for p in range(P)])
    sa = np.asarray(sqrt_ac, np.float64)[t].reshape(P, 1, 1, 1)
    sb = np.asarray(sqrt_1mac, np.float64)[t].reshape(P, 1, 1, 1)
    z = sa * y[None] + sb * eps
    target = eps if prediction == 'eps' else sa * eps - sb * y[None]
    return t, eps, np.tile(z, (H, 1, 1, 1)), np.tile(logsnr(t), H), target


def loss(out, target, H: int, P: int):
    """(L (H,), d_out (H P,S,S,3)): L_h = (1/P) sum_p mean (out_b - target_p)^2 and its gradient w.r.t. out."""
    out = np.asarray(out, np.float64).reshape(H, P, -1)
    r = out - np.asarray(target, np.float64).reshape(1, P, -1)
    n = r.shape[-1]
    return (r ** 2).sum((1, 2)) / (P * n), (2.0 / (P * n) * r).reshape(H * P, -1)


def hat(w) -> np.ndarray:
    w = np.asarray(w, np.float64)
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def tangent(dR, dt, R, t, P: int, translate: bool) -> np.ndarray:
    """(H, 3 or 6): g_omega = vee(N - N^T) with N = G_R R^T + g_t t^T, and g_delta = g_t, from the per-row dR (H P,3,3), dt."""
    H = len(R)
    G = np.asarray(dR, np.float64).reshape(H, P, 3, 3).sum(1)
    g = np.asarray(dt, np.float64).reshape(H, P, 3).sum(1)
    N = G @ np.swapaxes(np.asarray(R, np.float64), 1, 2) + g[:, :, None] * np.asarray(t, np.float64)[:, None, :]
    w = np.stack([N[:, 2, 1] - N[:, 1, 2], N[:, 0, 2] - N[:, 2, 0], N[:, 1, 0] - N[:, 0, 1]], -1)
    return np.concatenate([w, g], -1) if translate else w


def adam(grad, m, v, count: int, lr: float, b1=0.9, b2=0.999, eps=1e-8):
    """xunet_adam_step on a zero parameter buffer: (step, m, v) with step = -lr m_hat / (sqrt(v_hat) + eps)."""
    m = b1 * np.asarray(m, np.float64) + (1 - b1) * np.asarray(grad, np.float64)
    v = b2 * np.asarray(v, np.float64) + (1 - b2) * np.asarray(grad, np.float64) ** 2
    mh, vh = m / (1 - b1 ** count), v / (1 - b2 ** count)
    return -lr * mh / (np.sqrt(vh) + eps), m, v


def expm_so3(w) -> np.ndarray:
    """Rodrigues' formula with the kernel's small-angle branch."""
    w = np.asarray(w, np.float64)
    th2 = float(w @ w)
    if th2 < SMALL_ANGLE2:
        A, B = 1.0 - th2 / 6.0 + th2 * th2 / 120.0, 0.5 - th2 / 24.0 + th2 * th2 / 720.0
    else:
        th = math.sqrt(th2)
        A, B = math.sin(th) / th, 2.0 * math.sin(0.5 * th) ** 2 / th2
    return np.eye(3) + A * hat(w) + B * (np.outer(w, w) - th2 * np.eye(3))


def retract(step, R, t, translate: bool):
    """R_h <- exp([omega]x) R_h, t_h <- exp([omega]x) t_h + delta."""
    step = np.asarray(step, np.float64)
    E = np.stack([expm_so3(s[:3]) for s in step])
    tn = np.einsum('hij,hj->hi', E, np.asarray(t, np.float64))
    if translate:
        tn = tn + step[:, 3:6]
    return E @ np.asarray(R, np.float64), tn
