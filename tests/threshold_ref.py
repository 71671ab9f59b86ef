"""fp64 restatements of dynamic thresholding (Saharia et al. 2022, Imagen section 2.3): the per-view scale s as an order
statistic (a sort, then numpy's 'linear' interpolation written out), and the DDPM, DDIM and DPM-Solver++(2M) steps with
the per-view threshold in place of the fixed clip of tests/solver_ref.py (same formulas, same order of operations)."""
import math

import numpy as np
import torch

from tests import solver_ref as S


def quantile_linear(a, p: float) -> float:
    """np.quantile(a, p) of a 1-D array, method 'linear', in fp64: idx = (n - 1) p, lo = floor(idx), hi = min(lo + 1, n - 1),
    g = idx - lo, d = a[hi] - a[lo], q = a[lo] + d g if g < 0.5 else a[hi] - d (1 - g), on a sorted ascending."""
    a = np.sort(np.asarray(a, dtype=np.float64).ravel())
    n = a.size
    idx = (n - 1) * float(p)
    lo = int(math.floor(idx))
    hi = min(lo + 1, n - 1)
    g = idx - lo
    d = a[hi] - a[lo]
    return float(a[lo] + d * g) if g < 0.5 else float(a[hi] - d * (1.0 - g))


def threshold_scale(x0_view, p: float) -> np.float32:
    """The kernel's s of one view of fp32 values: max(fp32(quantile_p(|x0|)), 1)."""
    a = np.abs(np.asarray(x0_view, dtype=np.float32))
    return np.float32(max(np.float32(quantile_linear(a, p)), np.float32(1.0)))


def threshold(x0: torch.Tensor, p: float):
    """fp64 dynamic thresholding of x0 (B, ...) per view: s_b = max(1, quantile_p(|x0_b|)), x0_b <- clip(x0_b, -s_b, s_b) / s_b.
    Returns (x0, s) with s of shape (B,)."""
    flat = x0.reshape(x0.shape[0], -1)
    s = torch.tensor([max(1.0, quantile_linear(v.abs().numpy(), p)) for v in flat], dtype=torch.float64)
    sv = s.reshape((-1,) + (1,) * (x0.dim() - 1))
    return torch.maximum(torch.minimum(x0, sv), -sv) / sv, s


def guided_x0(eps_c, eps_u, z, ac, w, p):
    """The guided eps of sampling.py:133-134 and the unclipped x0 of :136, thresholded per view.  Returns (x0, s)."""
    eps = (1 + w) * eps_c - w * eps_u
    return threshold(math.sqrt(1. / ac) * z - math.sqrt(1. / ac - 1.) * eps, p)


def ddpm_step(eps_c, eps_u, z, ac, ac_next, noise, p, w=3.0):
    """One ancestral step (sampling.py:138-151) from alpha-bar ac to ac_next (1 after the last step, where sigma = 0):
    the posterior mean of the thresholded x0 plus sigma noise.  Returns (z_next, x0, s)."""
    x0, s = guided_x0(eps_c, eps_u, z, ac, w, p)
    beta = 1. - ac / ac_next
    c1 = beta * math.sqrt(ac_next) / (1. - ac)
    c2 = (1. - ac_next) * math.sqrt(1. - beta) / (1. - ac)
    sigma = 0.0 if ac_next >= 1.0 else math.exp(0.5 * math.log(max(beta * (1. - ac_next) / (1. - ac), 1e-20)))
    return c1 * x0 + c2 * z + sigma * noise, x0, s


def ddim_step(eps_c, eps_u, z, ac, ac_next, noise, p, eta=0.0, w=3.0):
    """solver_ref.ddim_step with the thresholded x0.  Returns (z_next, x0, s)."""
    x0, s = guided_x0(eps_c, eps_u, z, ac, w, p)
    eps = (z - math.sqrt(ac) * x0) / math.sqrt(1. - ac)
    sigma = eta * math.sqrt((1. - ac_next) / (1. - ac)) * math.sqrt(1. - ac / ac_next)
    z_next = math.sqrt(ac_next) * x0 + math.sqrt(max(1. - ac_next - sigma * sigma, 0.)) * eps + sigma * noise
    return z_next, x0, s


def dpmpp_2m_step(eps_c, eps_u, z, ac, ac_next, x0_prev, ac_prev, p, w=3.0):
    """solver_ref.dpmpp_2m_step with the thresholded x0 (x0_prev is the previous step's thresholded x0).
    Returns (z_next, x0, s)."""
    x0, s = guided_x0(eps_c, eps_u, z, ac, w, p)
    if ac_next >= 1.0:
        return x0.clone(), x0, s
    h = S._lam(ac_next) - S._lam(ac)
    d = x0
    if x0_prev is not None:
        r = (S._lam(ac) - S._lam(ac_prev)) / h
        d = (1. + 1. / (2. * r)) * x0 - (1. / (2. * r)) * x0_prev
    z_next = math.sqrt((1. - ac_next) / (1. - ac)) * z - math.sqrt(ac_next) * math.expm1(-h) * d
    return z_next, x0, s
