"""DDIM and DPM-Solver++(2M) on the GPU: the multistep step kernel against the fp64 steps of tests/solver_ref.py, an exact
denoiser driven through the step kernels, and the Sampler end to end on the tiny model against the oracle's forward."""
import numpy as np
import pytest
import torch

from oracle import xunet_ref as R
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200.sampling import Schedule, sampler_table
import novel_view_synthesis_3d_b200 as P
from tests import solver_ref as S
from tests.test_gpu_model import TINY, _pool_from_batch, _setup
from tests.util import np_batch, rel_l2

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def _step(lib, eps2, z, noise, n, w, tab, pos, seed, x0_hist, next_z2, next_logsnr2, b2):
    if x0_hist is None:
        rc = lib.xunet_sampler_step_table(eps2.data_ptr(), z.data_ptr(), noise, n, w, tab.data_ptr(), pos.data_ptr(),
                                          seed.data_ptr(), next_z2.data_ptr(), next_logsnr2.data_ptr(), b2, _stream())
    else:
        rc = lib.xunet_sampler_step_multistep(eps2.data_ptr(), z.data_ptr(), noise, n, w, tab.data_ptr(), pos.data_ptr(),
                                              seed.data_ptr(), x0_hist.data_ptr(), next_z2.data_ptr(),
                                              next_logsnr2.data_ptr(), b2, _stream())
    assert rc == 0, lib.xunet_last_error()
    pos.add_(1)


def test_multistep_kernel_matches_fp64_steps(lib):
    """Each step of a 6-row dpmpp_2m table with explicit eps: z against the fp64 step (fed the device's x0 history),
    x0_hist = the clipped x0, both halves of next_z2 = z, the row's log-SNR; a NaN history before the first step stays out."""
    sched = Schedule(6, spacing='logsnr')
    rows, _ = sampler_table(sched, 'dpmpp_2m', logsnr_lag=False)
    assert len(rows) == 6 and (rows[1:-1, 6] != 0).all()
    ac = S.alphas_cumprod()
    ts = list(sched.timesteps[::-1])
    g = torch.Generator().manual_seed(4)
    n, b2 = 2 * 8 * 8 * 3, 4
    tabd = torch.tensor(rows, dtype=torch.float64).float().cuda()
    noise = torch.randn(len(ts), n, generator=g, dtype=torch.float64)
    nd = noise.float().cuda()
    pos = torch.zeros(1, dtype=torch.int32, device='cuda')
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    hist = torch.full((n,), float('nan'), device='cuda')
    next_z2, next_logsnr2 = torch.zeros(2 * n, device='cuda'), torch.zeros(b2, device='cuda')
    for k, t in enumerate(ts):
        ec, eu, z = [torch.randn(n, generator=g, dtype=torch.float64) for _ in range(3)]
        ac_next = ac[ts[k + 1]] if k + 1 < len(ts) else 1.0
        prev = None if k == 0 else hist.double().cpu()
        ref, x0 = S.dpmpp_2m_step(ec, eu, z, ac[t], ac_next, prev, ac[ts[k - 1]] if k else None)
        eps2 = torch.cat([ec, eu]).float().cuda()
        zd = z.float().cuda()
        _step(lib, eps2, zd, nd.data_ptr(), n, 3.0, tabd, pos, seed, hist, next_z2, next_logsnr2, b2)
        assert bool(torch.isfinite(zd).all()) and bool(torch.isfinite(hist).all()), k
        # at t=999 sqrt(1/abar) ~ 6e4 amplifies fp32 rounding before the clip; compare on the clipped scale
        if t >= 998:
            assert float((zd.double().cpu() - ref).abs().max()) < 5e-3, k
            assert float((hist.double().cpu() - x0).abs().max()) < 5e-3, k
        else:
            assert rel_l2(zd, ref) < 1e-5, k
            assert rel_l2(hist, x0) < 1e-5, k
        assert torch.equal(next_z2[:n], zd) and torch.equal(next_z2[n:], zd)
        assert bool((next_logsnr2 == tabd[k, 5]).all())
    # the multistep entry point needs its history buffer
    assert lib.xunet_sampler_step_multistep(eps2.data_ptr(), zd.data_ptr(), None, n, 3.0, tabd.data_ptr(), pos.data_ptr(),
                                            seed.data_ptr(), None, next_z2.data_ptr(), next_logsnr2.data_ptr(), b2,
                                            _stream()) != 0


@pytest.mark.parametrize('method,steps,spacing', [('ddim', 50, 'linear'), ('dpmpp_2m', 25, 'logsnr')])
def test_exact_denoiser_on_the_device(lib, method, steps, spacing):
    """Exact eps of Gaussian data computed with torch on the device, the step kernel in between: the fp32 chain stays within
    1e-3 of the fp64 one on the CPU."""
    sched = Schedule(steps, spacing=spacing)
    rows, _ = sampler_table(sched, method)
    ac = S.alphas_cumprod()
    ts = list(sched.timesteps[::-1])
    n = 100_000
    z_T = torch.randn(n, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    ref = S.run_exact(method, sched.timesteps, z_T)
    tabd = torch.tensor(rows, dtype=torch.float64).float().cuda()
    pos = torch.zeros(1, dtype=torch.int32, device='cuda')
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    hist = torch.empty(n, device='cuda') if method == 'dpmpp_2m' else None
    next_z2, next_logsnr2 = torch.zeros(2 * n, device='cuda'), torch.zeros(2, device='cuda')
    z = z_T.float().cuda()
    for t in ts:
        e = S.exact_eps(z.double(), ac[t]).float()
        _step(lib, torch.cat([e, e]), z, None, n, 0.0, tabd, pos, seed, hist, next_z2, next_logsnr2, 2)
    err = float((z.double().cpu() - ref).abs().max())
    assert err <= 1e-3, err


def _oracle_chain(ref_params, rcfg, batch, B, method, ts, z0, noises, eta):
    """The oracle's forward plus the fp64 step, each forward fed the log-SNR of the timestep z is at."""
    ac = S.alphas_cumprod()
    z, x0 = z0, None
    for k, t in enumerate(ts):
        b = dict(batch, z=z, logsnr=torch.full((B,), float(R.logsnr_schedule_cosine(t / 1000.0)), dtype=torch.float64))
        ec = R.xunet_forward(ref_params, b, torch.ones(B), rcfg)
        eu = R.xunet_forward(ref_params, b, torch.zeros(B), rcfg)
        ac_next = ac[ts[k + 1]] if k + 1 < len(ts) else 1.0
        if method == 'ddim':
            z, x0 = S.ddim_step(ec, eu, z, ac[t], ac_next, noises[k], eta=eta)
        else:
            z, x0 = S.dpmpp_2m_step(ec, eu, z, ac[t], ac_next, x0, ac[ts[k - 1]] if k else None)
    return z


@pytest.mark.parametrize('method,eta', [('ddim', 0.5), ('dpmpp_2m', 0.0)])
def test_sampler_matches_oracle_loop(method, eta):
    """Six steps with explicit z_init and noise.  The schedule spans t = 700 .. 0: near t = 999, sqrt(1/abar) ~ 6e4 would
    amplify the fp32 forward's rounding before the clip, the reason the DDPM loop test runs the last timesteps only."""
    cfgd, S_, B = TINY, 16, 1
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S_, B, 'fp32')
    nb = np_batch(batch)
    ts = np.array([0, 50, 150, 300, 500, 700])
    g = torch.Generator().manual_seed(9)
    z0 = torch.randn(B, S_, S_, 3, generator=g, dtype=torch.float64)
    noises = [torch.randn(B, S_, S_, 3, generator=g, dtype=torch.float64) for _ in range(len(ts))]
    samp = P.Sampler(model, tree, B, S_, steps=6, w=3.0, method=method, eta=eta)
    samp.sched.timesteps, samp.sched.alphas_cumprod = ts, S.alphas_cumprod()[ts]
    out = samp.sample(nb, z_init=z0.numpy(), noises=[x.numpy() for x in noises])
    ref = _oracle_chain(ref_params, rcfg, batch, B, method, list(ts[::-1]), z0, noises, eta)
    assert rel_l2(out, ref) < 2e-3


def test_ddim_eta1_with_the_lag_reproduces_ddpm():
    cfgd, S_, B = TINY, 16, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S_, B, 'fp32', params='random')
    nb = np_batch(batch)
    a = P.Sampler(model, tree, B, S_, steps=6, w=3.0).sample(nb, seed=3)
    b = P.Sampler(model, tree, B, S_, steps=6, w=3.0, method='ddim', eta=1.0, logsnr_lag=True).sample(nb, seed=3)
    assert rel_l2(b, a) < 1e-4


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
def test_dpmpp_graph_replay_and_eager_are_bit_identical(dtype):
    """The multistep step in the captured graph, with the history buffer carried across replays and across two targets."""
    cfgd, S_, B = TINY, 16, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S_, B, dtype)
    nb = np_batch(batch)
    views, poses, K, tp = _pool_from_batch(nb)
    tp = {k: np.concatenate([tp[k], poses[k]], 1) for k in ('R', 't')}
    out = {}
    for use_graph in (True, False):
        samp = P.Sampler(model, tree, B, S_, steps=8, w=3.0, use_graph=use_graph, method='dpmpp_2m')
        out[use_graph] = (samp.sample(nb, seed=3), samp.sample_views(views, poses, K, tp, seed=3))
    assert torch.equal(out[True][0], out[False][0])
    assert torch.equal(out[True][1], out[False][1])
    assert bool(torch.isfinite(out[True][1]).all())


def test_dpmpp_stochastic_conditioning_reduces_to_sample():
    cfgd, S_, B = TINY, 16, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S_, B, 'fp32')
    nb = np_batch(batch)
    samp = P.Sampler(model, tree, B, S_, steps=8, w=3.0, method='dpmpp_2m')
    a = samp.sample(nb, seed=3)
    views, poses, K, tp = _pool_from_batch(nb)
    b = samp.sample_views(views, poses, K, tp, seed=3)
    assert rel_l2(b[:, 0], a) < 2e-3


def test_sampler_rejects_bad_arguments():
    model, _, _, tree, _, _ = _setup(TINY, 16, 1, 'fp32')
    for kw in (dict(method='euler'), dict(method='ddim', eta=2.0), dict(method='dpmpp_2m', eta=0.5),
               dict(spacing='cosine')):
        with pytest.raises(ValueError):
            P.Sampler(model, tree, 1, 16, steps=6, **kw)
    s = P.Sampler(model, tree, 1, 16, steps=10, method='dpmpp_2m')
    assert s.sched.timesteps[-1] == 999 and len(s.sched) == len(Schedule(10, spacing='logsnr')) and not s.logsnr_lag
