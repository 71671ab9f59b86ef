"""Dynamic thresholding on the GPU (xunet_sampler_step_dynamic): the per-view scale against the order-statistic restatement
of tests/threshold_ref.py bit for bit, the step against the fp64 threshold steps, the reduction to the static step's bits when
s = 1, the Sampler end to end on the tiny model against the oracle's forward, graph replay, and argument errors."""
import numpy as np
import pytest
import torch

from oracle import xunet_ref as R
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200.sampling import Schedule, sampler_table
import novel_view_synthesis_3d_b200 as P
from tests import solver_ref as S
from tests import threshold_ref as T
from tests.test_gpu_model import TINY, _pool_from_batch, _setup
from tests.util import np_batch, rel_l2

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _dyn(lib, eps2, z, noise, n, w, tab, pos, seed, x0_hist, B, p, scale, next_z2, next_logsnr2, b2):
    return lib.xunet_sampler_step_dynamic(_ptr(eps2), _ptr(z), _ptr(noise), n, w, _ptr(tab), _ptr(pos), _ptr(seed),
                                          _ptr(x0_hist), B, p, _ptr(scale), _ptr(next_z2), _ptr(next_logsnr2), b2, _stream())


def _static(lib, eps2, z, noise, n, w, tab, pos, seed, x0_hist, next_z2, next_logsnr2, b2):
    if x0_hist is None:
        return lib.xunet_sampler_step_table(_ptr(eps2), _ptr(z), _ptr(noise), n, w, _ptr(tab), _ptr(pos), _ptr(seed),
                                            _ptr(next_z2), _ptr(next_logsnr2), b2, _stream())
    return lib.xunet_sampler_step_multistep(_ptr(eps2), _ptr(z), _ptr(noise), n, w, _ptr(tab), _ptr(pos), _ptr(seed),
                                            _ptr(x0_hist), _ptr(next_z2), _ptr(next_logsnr2), b2, _stream())


def _views(kind, B, per, rng):
    """(B, per) fp32 inputs of one kind; the first view of the tied and the zeros kinds is degenerate (all equal / all 0)."""
    if kind == 'normal':
        return (rng.standard_normal((B, per)) * 3).astype(np.float32)
    if kind == 'tied':                       # x0 quantised to a few levels
        v = (np.round(rng.standard_normal((B, per)) * 1.5) * 0.75).astype(np.float32)
        v[0] = 2.5
        return v
    if kind == 'zeros':
        v = (rng.standard_normal((B, per)) * 2).astype(np.float32)
        v[rng.random((B, per)) < 0.6] = 0.0
        v[0] = 0.0
        return v
    return (rng.standard_normal((B, per)) * 10.0 ** rng.uniform(-6, 6, (B, per))).astype(np.float32)    # wide range


@pytest.mark.parametrize('kind', ['normal', 'tied', 'zeros', 'wide'])
@pytest.mark.parametrize('S_', [16, 64, 128, 256])
@pytest.mark.parametrize('B', [1, 3, 8])
def test_scale_is_the_order_statistic(lib, B, S_, kind):
    """A row with c_recip = 1, c_recipm1 = 0 makes the unclipped x0 exactly z; c_x0 = 1, c_z = sigma = 0 makes z' the
    thresholded x0.  scale_out equals the restatement on those values bit for bit, z' is clip(z, -s, s) / s in fp32, and s
    of a view is the same at every position of the batch."""
    per = S_ * S_ * 3
    n = B * per
    rng = np.random.default_rng(B * 1000 + S_)
    zv = _views(kind, B, per, rng)
    tab = torch.tensor([[1, 0, 1, 0, 0, 0.5, 0, 0]], dtype=torch.float32, device='cuda')
    pos = torch.zeros(1, dtype=torch.int32, device='cuda')
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    eps2 = torch.randn(2 * n, device='cuda')
    next_z2, next_logsnr2 = torch.empty(2 * n, device='cuda'), torch.empty(2 * B, device='cuda')
    for p in (0.995, 0.5, 1.0):
        got = {}
        for shift in ((0, 1) if B > 1 else (0,)):
            zs = np.roll(zv, shift, axis=0)
            z = torch.from_numpy(zs.reshape(-1).copy()).cuda()
            scale = torch.full((B,), float('nan'), device='cuda')
            assert _dyn(lib, eps2, z, None, n, 3.0, tab, pos, seed, None, B, p, scale, next_z2, next_logsnr2, 2 * B) == 0, \
                lib.xunet_last_error()
            s = scale.cpu().numpy()
            ref = np.array([T.threshold_scale(v, p) for v in zs], np.float32)
            assert s.tobytes() == ref.tobytes(), (p, shift, s, ref)
            expect = (np.clip(zs, -ref[:, None], ref[:, None]) / ref[:, None]).reshape(-1)
            assert np.array_equal(z.cpu().numpy(), expect), (p, shift)
            assert torch.equal(next_z2[:n], z) and torch.equal(next_z2[n:], z)
            assert bool((next_logsnr2 == 0.5).all())
            got[shift] = s
        if B > 1:
            assert np.roll(got[0], 1).tobytes() == got[1].tobytes()
        if kind in ('tied', 'zeros'):
            assert got[0][0] == (2.5 if kind == 'tied' else 1.0)


@pytest.mark.parametrize('method,eta,spacing', [('ddpm', 0.0, 'linear'), ('ddim', 0.5, 'linear'), ('dpmpp_2m', 0.0, 'logsnr')])
def test_step_matches_fp64_threshold_steps(lib, method, eta, spacing):
    """Each step of a 6-row table with explicit eps (w = 3, so x0 leaves [-1, 1] and s > 1 at high t): z against the fp64
    threshold step (fed the device's x0 history), the thresholded x0 in x0_hist, s, both halves of next_z2 and the row's
    log-SNR; the dpmpp history starts NaN-filled."""
    sched = Schedule(6, spacing=spacing)
    rows, _ = sampler_table(sched, method, eta=eta, logsnr_lag=False)
    ac = S.alphas_cumprod()
    ts = list(sched.timesteps[::-1])
    g = torch.Generator().manual_seed(6)
    B, per = 2, 8 * 8 * 3
    n, b2 = B * per, 2 * B
    tabd = torch.tensor(rows, dtype=torch.float64).float().cuda()
    noise = torch.randn(len(ts), n, generator=g, dtype=torch.float64)
    nd = noise.float().cuda()
    pos = torch.zeros(1, dtype=torch.int32, device='cuda')
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    hist = torch.full((n,), float('nan'), device='cuda') if method == 'dpmpp_2m' else None
    scale = torch.zeros(B, device='cuda')
    next_z2, next_logsnr2 = torch.zeros(2 * n, device='cuda'), torch.zeros(b2, device='cuda')
    saw_big = False
    for k, t in enumerate(ts):
        ec, eu, z = [torch.randn(B, per, generator=g, dtype=torch.float64) for _ in range(3)]
        ac_next = ac[ts[k + 1]] if k + 1 < len(ts) else 1.0
        nk = noise[k].reshape(B, per)
        if method == 'ddpm':
            ref, x0, s = T.ddpm_step(ec, eu, z, ac[t], ac_next, nk, 0.995)
        elif method == 'ddim':
            ref, x0, s = T.ddim_step(ec, eu, z, ac[t], ac_next, nk, 0.995, eta=eta)
        else:
            prev = None if k == 0 else hist.double().cpu().reshape(B, per)
            ref, x0, s = T.dpmpp_2m_step(ec, eu, z, ac[t], ac_next, prev, ac[ts[k - 1]] if k else None, 0.995)
        eps2 = torch.cat([ec.reshape(-1), eu.reshape(-1)]).float().cuda()
        zd = z.reshape(-1).float().cuda()
        assert _dyn(lib, eps2, zd, nd, n, 3.0, tabd, pos, seed, hist, B, 0.995, scale, next_z2, next_logsnr2, b2) == 0, \
            lib.xunet_last_error()
        pos.add_(1)
        assert bool(torch.isfinite(zd).all()), k
        assert float((scale.double().cpu() - s).abs().max()) <= 1e-5 * float(s.max()), (k, scale, s)
        saw_big |= bool((s > 1.5).any())
        if t >= 998:          # sqrt(1/abar) ~ 6e4 amplifies fp32 rounding before the threshold
            assert float((zd.double().cpu() - ref.reshape(-1)).abs().max()) < 5e-3, k
        else:
            assert rel_l2(zd, ref) < 1e-5, k
        if hist is not None:
            assert bool(torch.isfinite(hist).all()), k
            assert rel_l2(hist, x0) < 1e-5, k
        assert torch.equal(next_z2[:n], zd) and torch.equal(next_z2[n:], zd)
        assert bool((next_logsnr2 == tabd[k, 5]).all())
    assert saw_big


@pytest.mark.parametrize('method,explicit_noise', [('ddim', True), ('ddim', False), ('dpmpp_2m', True), ('dpmpp_2m', False)])
def test_views_with_unit_scale_get_the_static_bits(lib, method, explicit_noise):
    """A batch mixing views whose x0 stays inside [-1, 1] (s = 1) with views far outside it: the s = 1 views come out
    bit-identical to xunet_sampler_step_table / _multistep (z, both halves of next_z2, x0_hist), the others do not."""
    if method == 'ddim':
        rows, _ = sampler_table(Schedule(25), 'ddim', eta=0.5)
        k = 18
    else:
        rows, _ = sampler_table(Schedule(25, spacing='logsnr'), 'dpmpp_2m')
        k = 10
        assert rows[k, 6] != 0.0
    tab = torch.tensor(rows, dtype=torch.float64).float().cuda()
    c_recip, c_recipm1 = float(tab[k, 0]), float(tab[k, 1])
    B, per = 4, 16 * 16 * 3
    n, b2 = B * per, 2 * B
    g = torch.Generator().manual_seed(11)
    e = torch.randn(B, per, generator=g)
    x0t = torch.rand(B, per, generator=g) * 2 - 1
    x0t[0::2] *= 0.9          # views 0, 2: |x0| <= 0.9 -> s = 1
    x0t[1::2] *= 4.0          # views 1, 3: s ~ 4
    z0 = ((x0t + c_recipm1 * e) / c_recip).reshape(-1).cuda()
    eps2 = torch.cat([e.reshape(-1), e.reshape(-1)]).cuda()
    noise = torch.randn(len(rows), n, generator=g).cuda() if explicit_noise else None
    seed = torch.tensor([987654321], dtype=torch.int64, device='cuda')
    hist0 = torch.randn(n, generator=g).cuda() if method == 'dpmpp_2m' else None
    out = {}
    for dyn in (False, True):
        z = z0.clone()
        hist = None if hist0 is None else hist0.clone()
        pos = torch.full((1,), k, dtype=torch.int32, device='cuda')
        next_z2, next_logsnr2 = torch.zeros(2 * n, device='cuda'), torch.zeros(b2, device='cuda')
        scale = torch.zeros(B, device='cuda')
        if dyn:
            rc = _dyn(lib, eps2, z, noise, n, 3.0, tab, pos, seed, hist, B, 0.995, scale, next_z2, next_logsnr2, b2)
        else:
            rc = _static(lib, eps2, z, noise, n, 3.0, tab, pos, seed, hist, next_z2, next_logsnr2, b2)
        assert rc == 0, lib.xunet_last_error()
        out[dyn] = (z.reshape(B, per), next_z2.reshape(2, B, per), next_logsnr2,
                    None if hist is None else hist.reshape(B, per), scale.cpu())
    (zs, nzs, ls, hs, _), (zd, nzd, ld, hd, sd) = out[False], out[True]
    assert sd[0] == 1.0 and sd[2] == 1.0 and bool((sd[1::2] > 3.0).all()), sd
    assert torch.equal(ld, ls)
    for v in (0, 2):
        assert torch.equal(zd[v], zs[v]) and torch.equal(nzd[:, v], nzs[:, v]), v
        if hd is not None:
            assert torch.equal(hd[v], hs[v]), v
    for v in (1, 3):
        assert not torch.equal(zd[v], zs[v]), v


def _oracle_chain(ref_params, rcfg, batch, B, method, ts, z0, noises, eta, p):
    """The oracle's forward plus the fp64 threshold step, each forward fed the log-SNR of the timestep z is at."""
    ac = S.alphas_cumprod()
    z, x0 = z0, None
    for k, t in enumerate(ts):
        b = dict(batch, z=z, logsnr=torch.full((B,), float(R.logsnr_schedule_cosine(t / 1000.0)), dtype=torch.float64))
        ec = R.xunet_forward(ref_params, b, torch.ones(B), rcfg)
        eu = R.xunet_forward(ref_params, b, torch.zeros(B), rcfg)
        ac_next = ac[ts[k + 1]] if k + 1 < len(ts) else 1.0
        if method == 'ddim':
            z, x0, _ = T.ddim_step(ec, eu, z, ac[t], ac_next, noises[k], p, eta=eta)
        else:
            z, x0, _ = T.dpmpp_2m_step(ec, eu, z, ac[t], ac_next, x0, ac[ts[k - 1]] if k else None, p)
    return z


@pytest.mark.parametrize('method,eta', [('ddim', 0.5), ('dpmpp_2m', 0.0)])
def test_sampler_matches_oracle_loop(method, eta):
    """Six steps with explicit z_init and noise over t = 700 .. 0 (as tests/test_gpu_sampler_solvers.py), two views: the
    thresholded sampler against the oracle's forward plus the fp64 threshold step.  It differs from the static sampler."""
    cfgd, S_, B = TINY, 16, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S_, B, 'fp32')
    nb = np_batch(batch)
    ts = np.array([0, 50, 150, 300, 500, 700])
    g = torch.Generator().manual_seed(9)
    z0 = torch.randn(B, S_, S_, 3, generator=g, dtype=torch.float64)
    noises = [torch.randn(B, S_, S_, 3, generator=g, dtype=torch.float64) for _ in range(len(ts))]
    outs = {}
    for p in (None, 0.995):
        samp = P.Sampler(model, tree, B, S_, steps=6, w=3.0, method=method, eta=eta, dynamic_threshold=p)
        samp.sched.timesteps, samp.sched.alphas_cumprod = ts, S.alphas_cumprod()[ts]
        outs[p] = samp.sample(nb, z_init=z0.numpy(), noises=[x.numpy() for x in noises])
    ref = _oracle_chain(ref_params, rcfg, batch, B, method, list(ts[::-1]), z0, noises, eta, 0.995)
    assert rel_l2(outs[0.995], ref) < 2e-3
    assert rel_l2(outs[0.995], outs[None]) > 1e-2


@pytest.mark.parametrize('method,dtype', [('ddpm', 'bf16'), ('dpmpp_2m', 'fp32')])
def test_graph_replay_and_eager_are_bit_identical(method, dtype):
    cfgd, S_, B = TINY, 16, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S_, B, dtype)
    nb = np_batch(batch)
    views, poses, K, tp = _pool_from_batch(nb)
    tp = {k: np.concatenate([tp[k], poses[k]], 1) for k in ('R', 't')}
    out = {}
    for use_graph in (True, False):
        samp = P.Sampler(model, tree, B, S_, steps=8, w=3.0, use_graph=use_graph, method=method, dynamic_threshold=0.995)
        out[use_graph] = (samp.sample(nb, seed=3), samp.sample_views(views, poses, K, tp, seed=3))
    assert torch.equal(out[True][0], out[False][0])
    assert torch.equal(out[True][1], out[False][1])
    assert bool(torch.isfinite(out[True][1]).all())


def test_argument_errors(lib):
    B, per = 2, 48
    n = B * per
    f = lambda m: torch.zeros(m, device='cuda')
    eps2, z, tab, nz2, nl2, hist, scale = f(2 * n), f(n), f(8), f(2 * n), f(2 * B), f(n), f(B)
    pos = torch.zeros(1, dtype=torch.int32, device='cuda')
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    good = dict(eps2=eps2, z=z, noise=None, n=n, w=3.0, tab=tab, pos=pos, seed=seed, x0_hist=None, B=B, p=0.995, scale=scale,
                next_z2=nz2, next_logsnr2=nl2, b2=2 * B)
    call = lambda **kw: _dyn(lib, **{**good, **kw})
    assert call() == 0, lib.xunet_last_error()
    assert call(x0_hist=hist, scale=None, p=1.0) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    bad = [dict(eps2=None), dict(z=None), dict(tab=None), dict(pos=None), dict(seed=None), dict(next_z2=None),
           dict(next_logsnr2=None), dict(n=0), dict(b2=0), dict(B=0), dict(B=-1), dict(B=5), dict(n=n - 1),
           dict(n=_lib.SAMPLER_DYN_MAX_PER + 1, B=1), dict(p=0.0), dict(p=-0.5), dict(p=1.0 + 1e-12), dict(p=float('nan')),
           dict(p=float('inf'))]
    for kw in bad:
        assert call(**kw) != 0, kw
        assert lib.xunet_last_error(), kw
    assert call(n=_lib.SAMPLER_DYN_MAX_PER + 1, B=1) != 0
    assert b'XUNET_SAMPLER_DYN_MAX_PER' in lib.xunet_last_error()
