"""fp64 restatements of the DDIM and DPM-Solver++(2M) sampler steps, written from the papers' formulas in alpha-bar (not from
the device table, which the tests check against them), and the exact denoiser of Gaussian data the convergence tests use."""
import math

import numpy as np
import torch

from oracle import xunet_ref as R


def _guided_x0(eps_c, eps_u, z, ac, w):
    """The guided eps of sampling.py:133-134 and the clipped x0 of :136-137, at alpha-bar ac."""
    eps = (1 + w) * eps_c - w * eps_u
    return torch.clamp(math.sqrt(1. / ac) * z - math.sqrt(1. / ac - 1.) * eps, -1., 1.)


def ddim_step(eps_c, eps_u, z, ac, ac_next, noise, eta=0.0, w=3.0):
    """One DDIM step (Song et al. 2021, eq. 12 and 16) from alpha-bar ac to ac_next (1 after the last step), with eps
    re-derived from the clipped x0 (as guided-diffusion does).  Returns (z_next, x0)."""
    x0 = _guided_x0(eps_c, eps_u, z, ac, w)
    eps = (z - math.sqrt(ac) * x0) / math.sqrt(1. - ac)
    sigma = eta * math.sqrt((1. - ac_next) / (1. - ac)) * math.sqrt(1. - ac / ac_next)
    z_next = math.sqrt(ac_next) * x0 + math.sqrt(max(1. - ac_next - sigma * sigma, 0.)) * eps + sigma * noise
    return z_next, x0


def _lam(ac):
    return 0.5 * (math.log(ac) - math.log(1. - ac))          # log(alpha / sigma)


def dpmpp_2m_step(eps_c, eps_u, z, ac, ac_next, x0_prev=None, ac_prev=None, w=3.0):
    """One step of DPM-Solver++(2M) (Lu et al. 2022, Algorithm 2) from alpha-bar ac to ac_next, in data prediction with
    the clipped x0: z' = (sigma'/sigma) z - alpha' (e^-h - 1) D, D = (1 + 1/2r) x0 - (1/2r) x0_prev, r = h_prev / h.
    Without x0_prev / ac_prev, and on the last step (ac_next = 1, where it returns x0), the step is first order.
    Returns (z_next, x0)."""
    x0 = _guided_x0(eps_c, eps_u, z, ac, w)
    if ac_next >= 1.0:
        return x0.clone(), x0
    h = _lam(ac_next) - _lam(ac)
    d = x0
    if x0_prev is not None:
        r = (_lam(ac) - _lam(ac_prev)) / h
        d = (1. + 1. / (2. * r)) * x0 - (1. / (2. * r)) * x0_prev
    z_next = math.sqrt((1. - ac_next) / (1. - ac)) * z - math.sqrt(ac_next) * math.expm1(-h) * d
    return z_next, x0


def alphas_cumprod():
    return R.schedule_tables()['alphas_cumprod']


# ---- the exact denoiser of per-pixel Gaussian data x0 ~ N(mu, s^2) ------------------------------------------------------
MU, SD = 0.1, 0.2


def exact_eps(z, ac, mu=MU, s=SD):
    """eps_hat = E[eps | z] for z = sqrt(ac) x0 + sqrt(1 - ac) eps."""
    a, sg2 = math.sqrt(ac), 1. - ac
    x0 = mu + a * s * s * (z - a * mu) / (ac * s * s + sg2)
    return (z - a * x0) / math.sqrt(sg2)


def ode_endpoint(z_T, ac_T, mu=MU, s=SD):
    """The probability-flow ODE's x0 from z_T at alpha-bar ac_T."""
    return mu + s * (z_T - math.sqrt(ac_T) * mu) / math.sqrt(ac_T * s * s + 1. - ac_T)


def run_exact(method, timesteps, z_T, *, eta=0.0, noises=None):
    """The chain over `timesteps` (ascending, as Schedule.timesteps) with the exact eps (guidance w = 0), in fp64 through
    the steps above.  Returns the final z."""
    ac_full = alphas_cumprod()
    ts = list(np.asarray(timesteps)[::-1])
    z, x0_prev = z_T, None
    for k, t in enumerate(ts):
        ac, ac_next = ac_full[t], (ac_full[ts[k + 1]] if k + 1 < len(ts) else 1.0)
        e = exact_eps(z, ac)
        if method == 'ddim':
            z, _ = ddim_step(e, e, z, ac, ac_next, 0. if noises is None else noises[k], eta=eta, w=0.0)
        else:
            z, x0 = dpmpp_2m_step(e, e, z, ac, ac_next, x0_prev, ac_full[ts[k - 1]] if k > 0 else None, w=0.0)
            x0_prev = x0
    return z
