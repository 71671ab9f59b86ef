"""The DDIM and DPM-Solver++(2M) tables of `sampler_table` (no GPU): DDIM at eta = 1 is the DDPM posterior, the last and the
first-order rows, log-SNR spacing, the table against the fp64 steps of tests/solver_ref.py, and convergence on an exact
denoiser of Gaussian data, where the probability-flow ODE has a closed-form endpoint."""
import math

import numpy as np
import pytest
import torch

from novel_view_synthesis_3d_b200.sampling import METHODS, Schedule, logsnr_schedule_cosine, sampler_table
from tests import solver_ref as S

C_RECIP, C_RECIPM1, C_X0, C_Z, SIGMA, LOGSNR, C_PREV = range(7)


def table_step(row, eps_c, eps_u, z, x0_prev, noise, w=3.0):
    """The step kernel's formula on one table row, in fp64: returns (z_next, x0)."""
    eps = (1 + w) * eps_c - w * eps_u
    x0 = torch.clamp(row[C_RECIP] * z - row[C_RECIPM1] * eps, -1., 1.)
    z_next = row[C_X0] * x0 + row[C_Z] * z + row[SIGMA] * noise
    if row[C_PREV] != 0.0:
        z_next = z_next + row[C_PREV] * x0_prev
    return z_next, x0


@pytest.mark.parametrize('steps', [1000, 256, 25])
def test_ddim_eta1_is_the_ddpm_posterior(steps):
    sched = Schedule(steps)
    ddpm, l0 = sampler_table(sched, 'ddpm')
    ddim, l1 = sampler_table(sched, 'ddim', eta=1.0, logsnr_lag=True)
    # the ddpm rows form beta = 1 - abar/abar', alpha = 1 - beta and 1 - abar by subtraction, and so lose up to
    # log10(1/alpha), log10(1/beta) and log10(1/(1 - abar)) digits (alpha ~ 4e-5 on the first row); ddim does not
    i = np.arange(len(sched) - 1, -1, -1)
    alpha, ac = sched.alphas_cumprod[i] / sched.alphas_cumprod_prev[i], sched.alphas_cumprod[i]
    rtol = 1e-12 + 8 * np.finfo(np.float64).eps * (1 / alpha + 1 / np.maximum(1 - alpha, 1e-300) + 1 / (1 - ac))
    for c in (C_X0, C_Z, SIGMA):
        err = np.abs(ddim[:, c] - ddpm[:, c])
        assert (err <= rtol * np.abs(ddpm[:, c])).all(), (c, np.argmax(err / rtol / np.abs(ddpm[:, c]).clip(1e-300)))
    assert float(np.median(np.abs(ddim[:-1, C_X0:SIGMA + 1] / ddpm[:-1, C_X0:SIGMA + 1] - 1))) < 1e-14
    assert np.array_equal(ddim[:, LOGSNR], ddpm[:, LOGSNR]) and l0 == l1 == -20.0
    assert np.array_equal(ddim[:, [C_RECIP, C_RECIPM1]], ddpm[:, [C_RECIP, C_RECIPM1]])


def test_ddpm_rows_are_the_reference_posterior():
    """The default table: the schedule's posterior tables, sigma 0 at t = 0, the lagging log-SNR, no c_prev."""
    sched = Schedule(256)
    rows, first = sampler_table(sched)
    i = np.arange(len(sched) - 1, -1, -1)
    assert np.array_equal(rows[:, C_X0], sched.posterior_mean_coef1[i]) and np.array_equal(rows[:, C_Z], sched.posterior_mean_coef2[i])
    assert np.array_equal(rows[:, SIGMA], np.where(i == 0, 0.0, np.exp(0.5 * sched.posterior_log_variance_clipped[i])))
    assert np.array_equal(rows[:, LOGSNR], logsnr_schedule_cosine(sched.timesteps[i] / 1000.0)) and first == -20.0
    assert not rows[:, C_PREV:].any()


@pytest.mark.parametrize('method,eta', [('ddpm', 0.0), ('ddim', 0.0), ('ddim', 0.5), ('ddim', 1.0), ('dpmpp_2m', 0.0)])
@pytest.mark.parametrize('spacing', ['linear', 'logsnr'])
def test_last_row_returns_x0(method, eta, spacing):
    rows, _ = sampler_table(Schedule(25, spacing=spacing), method, eta=eta)
    assert np.isfinite(rows).all()
    assert rows[-1, C_X0] == 1.0 and rows[-1, C_Z] == 0.0 and rows[-1, C_PREV] == 0.0 and rows[-1, SIGMA] == 0.0


@pytest.mark.parametrize('steps,spacing', [(25, 'logsnr'), (50, 'logsnr'), (50, 'linear'), (1000, 'linear')])
def test_dpmpp_rows_reduce_to_ddim(steps, spacing):
    """First-order rows (the first and the last) are DDIM at eta = 0, and in every row c_x0 + c_prev is DDIM's c_x0: with a
    constant x0 the solver is DDIM."""
    sched = Schedule(steps, spacing=spacing)
    dpm, _ = sampler_table(sched, 'dpmpp_2m')
    ddim, _ = sampler_table(sched, 'ddim', eta=0.0)
    first = dpm[:, C_PREV] == 0.0
    assert first[0] and first[-1] and not first[1:-1].any()
    np.testing.assert_allclose(dpm[first][:, :6], ddim[first][:, :6], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(dpm[:, C_X0] + dpm[:, C_PREV], ddim[:, C_X0], rtol=1e-10, atol=1e-15)
    np.testing.assert_allclose(dpm[:, C_Z], ddim[:, C_Z], rtol=1e-12, atol=0)
    assert not dpm[:, SIGMA].any()


@pytest.mark.parametrize('steps,count', [(10, 9), (25, 19), (50, 36), (100, 65), (256, 142), (1000, None)])
def test_logsnr_spacing(steps, count):
    sched = Schedule(steps, spacing='logsnr')
    ts = sched.timesteps[::-1]
    assert ts[0] == 999 and ts[-1] == 0 and (np.diff(ts) < 0).all() and len(sched) <= steps
    if count is not None:
        assert len(sched) == count
    ac = S.alphas_cumprod()
    np.testing.assert_array_equal(sched.alphas_cumprod, ac[sched.timesteps])


@pytest.mark.parametrize('method', ['ddpm', 'ddim', 'dpmpp_2m'])
def test_unlagged_logsnr(method):
    sched = Schedule(25, spacing='logsnr')
    rows, first = sampler_table(sched, method, logsnr_lag=False)
    t = sched.timesteps[::-1] / 1000.0
    assert first == float(logsnr_schedule_cosine(t[0]))
    np.testing.assert_array_equal(rows[:-1, LOGSNR], logsnr_schedule_cosine(t[1:]))


def test_bad_arguments_are_rejected():
    sched = Schedule(10)
    for kw in (dict(method='euler'), dict(method='ddim', eta=1.5), dict(method='ddim', eta=-0.1),
               dict(method='ddim', eta=float('nan')), dict(method='ddpm', eta=0.5), dict(method='dpmpp_2m', eta=0.1)):
        with pytest.raises(ValueError):
            sampler_table(sched, kw.pop('method'), **kw)
    with pytest.raises(ValueError):
        Schedule(10, spacing='quadratic')
    assert METHODS == ('ddpm', 'ddim', 'dpmpp_2m')


@pytest.mark.parametrize('method,eta,steps,spacing', [('ddim', 0.0, 25, 'linear'), ('ddim', 0.5, 25, 'linear'),
                                                       ('ddim', 1.0, 10, 'logsnr'), ('dpmpp_2m', 0.0, 25, 'logsnr'),
                                                       ('dpmpp_2m', 0.0, 50, 'linear')])
def test_table_matches_fp64_steps(method, eta, steps, spacing):
    """The kernel's formula on the table, in fp64, equals stepping with the papers' formulas in alpha-bar."""
    sched = Schedule(steps, spacing=spacing)
    rows, _ = sampler_table(sched, method, eta=eta)
    ac = S.alphas_cumprod()
    ts = list(sched.timesteps[::-1])
    g = torch.Generator().manual_seed(5)
    n = 4096
    z = torch.randn(n, generator=g, dtype=torch.float64)
    zt, x0t, x0r = z.clone(), None, None
    for k, t in enumerate(ts):
        ec, eu, nz = (torch.randn(n, generator=g, dtype=torch.float64) * 0.3 for _ in range(3))
        ac_next = ac[ts[k + 1]] if k + 1 < len(ts) else 1.0
        zt, x0t = table_step(rows[k], ec, eu, zt, x0t, nz)
        if method == 'ddim':
            z, x0r = S.ddim_step(ec, eu, z, ac[t], ac_next, nz, eta=eta)
        else:
            z, x0r = S.dpmpp_2m_step(ec, eu, z, ac[t], ac_next, x0r, ac[ts[k - 1]] if k else None)
        assert float((zt - z).abs().max()) <= 1e-12 * max(1.0, float(z.abs().max())), (k, t)


def _rms_exact(method, steps, spacing):
    sched = Schedule(steps, spacing=spacing)
    z_T = torch.randn(100_000, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    out = S.run_exact(method, sched.timesteps, z_T)
    ref = S.ode_endpoint(z_T, S.alphas_cumprod()[999])
    return float(((out - ref) ** 2).mean().sqrt())


def test_exact_denoiser_convergence():
    """DDIM is first order in the step; DPM-Solver++(2M) on log-SNR spacing reaches 256-step DDIM's error in 36 forwards."""
    d50, d100, d256 = (_rms_exact('ddim', s, 'linear') for s in (50, 100, 256))
    assert 1.8 <= d50 / d100 <= 2.2, (d50, d100)
    p25, p50 = (_rms_exact('dpmpp_2m', s, 'logsnr') for s in (25, 50))
    assert p25 <= 6e-3, p25
    assert p50 < d256, (p50, d256)
    assert math.isfinite(p25) and p50 < p25
