"""Autoguidance (Karras et al. 2024) on the GPU: `Sampler(guide_params=...)` and `xunet_sampler_step_guide`.

The bit-exact checks rest on two fp32 identities that hold whether or not nvcc contracts (1+w) a - w b to an fma:
1 a - 0 b = a (w = 0, any guide) and 2 a - a = a (a guide equal to the model, w = 1).  A distinct guide, of other params or
a narrower config, is checked against a host loop of model.apply / guide.apply and the fp64 steps of tests/solver_ref.py."""
import math

import numpy as np
import pytest
import torch

from oracle import xunet_ref as R
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200.sampling import Schedule, sampler_table
import novel_view_synthesis_3d_b200 as P
from tests import solver_ref as SR
from tests.test_gpu_model import SMALL, THREE, TINY, _setup
from tests.util import np_batch, rel_l2, to_ref_cfg

pytestmark = pytest.mark.gpu

TINY64 = dict(TINY, ch=64)       # the main model of the narrow-guide cases: TINY is the same topology at half the width


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _random_params(cfgd, S, seed):
    return R.init_params(to_ref_cfg(P.XUNet(**cfgd).config), S, seed=seed, zero_init=False, bias_std=0.1)


def _two_view_pool(B, S):
    """2 source views and 2 target poses from two synthetic batches."""
    a, b = (np_batch(R.synthetic_batch(B, S, seed=s)[0]) for s in (1234, 4321))
    views = np.stack([a['x'], b['x']], 1)
    poses = {'R': np.stack([a['R1'], b['R1']], 1), 't': np.stack([a['t1'], b['t1']], 1)}
    targets = {'R': np.stack([a['R2'], b['R2']], 1), 't': np.stack([a['t2'], b['t2']], 1)}
    return views, poses, a['K'], targets


# ---- 1. w = 0: any guide gives the unguided bits --------------------------------------------------------------------------
@pytest.mark.parametrize('prediction', ['eps', 'v'])
@pytest.mark.parametrize('dynamic', [None, 0.9])
@pytest.mark.parametrize('method,eta', [('ddpm', 0.0), ('ddim', 0.5), ('dpmpp_2m', 0.0), ('consistency', 0.0)])
def test_w0_with_any_guide_is_the_unguided_sampler(method, eta, dynamic, prediction):
    S, B = 16, 2
    model, _, _, tree, batch, _ = _setup(TINY64, S, B, 'fp32', params='random')
    nb = np_batch(batch)
    kw = dict(steps=6, method=method, eta=eta, dynamic_threshold=dynamic, prediction=prediction)
    ref = P.Sampler(model, tree, B, S, w=None, **kw).sample(nb, seed=5)
    guide = P.XUNet(**TINY, dtype='fp32')
    samp = P.Sampler(model, tree, B, S, w=0.0, guide_params=_random_params(TINY, S, 8), guide_model=guide, **kw)
    out = samp.sample(nb, seed=5)
    assert bool(torch.isfinite(ref).all())
    assert torch.equal(out, ref)


# ---- 2. a guide equal to the model at w = 1 -------------------------------------------------------------------------------
SELF_CASES = [(TINY, 16, 2, 'fp32'), (SMALL, 64, 2, 'bf16')]
SELF_IDS = ['tiny16-fp32', 'small64-bf16']


@pytest.mark.parametrize('cfgd,S,B,dtype', SELF_CASES, ids=SELF_IDS)
@pytest.mark.parametrize('method', ['ddpm', 'dpmpp_2m'])
def test_self_guide_at_w1_is_the_unguided_sampler(cfgd, S, B, dtype, method):
    model, _, _, tree, batch, _ = _setup(cfgd, S, B, dtype, params='random')
    nb = np_batch(batch)
    views, poses, K, targets = _two_view_pool(B, S)
    for cache in (dict(), dict(cache_interval=3, cache_level=1)):
        kw = dict(steps=8, method=method, **cache)
        plain = P.Sampler(model, tree, B, S, w=None, **kw)
        ref = plain.sample(nb, seed=3)
        ref_v, ref_c = plain.sample_views(views, poses, K, targets, seed=3, return_choices=True)
        samp = P.Sampler(model, tree, B, S, w=1.0, guide_params=tree, **kw)
        # the guide runs on its own engine, with its own workspace and output
        assert samp.eng is model.engine(B, S, False) and samp.guide_eng is not samp.eng
        assert samp.guide_eng.eps.data_ptr() != samp.eng.eps.data_ptr()
        out = samp.sample(nb, seed=3)
        out_v, out_c = samp.sample_views(views, poses, K, targets, seed=3, return_choices=True)
        assert bool(torch.isfinite(ref_v).all())
        assert torch.equal(out, ref), cache
        assert np.array_equal(out_c, ref_c) and len(set(ref_c.ravel())) > 1, cache
        assert torch.equal(out_v, ref_v), cache


# ---- 3. a distinct guide against a host loop in fp64 ----------------------------------------------------------------------
def _host_chain(model, params, guide, guide_params, nb, B, method, ts, z0, noises, eta, w):
    """model.apply and guide.apply on the current z, the outputs combined and stepped in fp64 (tests/solver_ref.py); each
    forward is fed the log-SNR of the timestep z is at."""
    ac = SR.alphas_cumprod()
    z, x0 = z0, None
    ones = np.ones(B, np.float32)
    for k, t in enumerate(ts):
        b = dict(nb, z=z.numpy(), logsnr=np.full((B,), float(R.logsnr_schedule_cosine(t / 1000.0))))
        a = model.apply({'params': params}, b, cond_mask=ones, train=False).double().cpu()
        g = guide.apply({'params': guide_params}, b, cond_mask=ones, train=False).double().cpu()
        ac_next = ac[ts[k + 1]] if k + 1 < len(ts) else 1.0
        if method == 'ddim':
            z, x0 = SR.ddim_step(a, g, z, ac[t], ac_next, noises[k], eta=eta, w=w)
        else:
            z, x0 = SR.dpmpp_2m_step(a, g, z, ac[t], ac_next, x0, ac[ts[k - 1]] if k else None, w=w)
    return z


@pytest.mark.parametrize('guide_kind', ['params', 'narrow'])
@pytest.mark.parametrize('method,eta', [('ddim', 0.5), ('dpmpp_2m', 0.0)])
def test_distinct_guide_matches_the_host_loop(guide_kind, method, eta):
    S, B, w = 16, 2, 2.0
    model, _, _, tree, batch, _ = _setup(TINY64, S, B, 'fp32', params='random')
    nb = np_batch(batch)
    if guide_kind == 'narrow':
        guide, gparams = P.XUNet(**TINY, dtype='fp32'), _random_params(TINY, S, 8)
    else:
        guide, gparams = model, _random_params(TINY64, S, 8)
    ts = np.array([0, 50, 150, 300, 500, 700])
    g = torch.Generator().manual_seed(9)
    z0 = torch.randn(B, S, S, 3, generator=g, dtype=torch.float64)
    noises = [torch.randn(B, S, S, 3, generator=g, dtype=torch.float64) for _ in range(len(ts))]
    samp = P.Sampler(model, tree, B, S, steps=6, w=w, method=method, eta=eta, guide_params=gparams,
                     guide_model=None if guide is model else guide)
    samp.sched.timesteps, samp.sched.alphas_cumprod = ts, SR.alphas_cumprod()[ts]
    out = samp.sample(nb, z_init=z0.numpy(), noises=[x.numpy() for x in noises])
    ref = _host_chain(model, tree, guide, gparams, nb, B, method, list(ts[::-1]), z0, noises, eta, w)
    # the guide's contribution is not negligible: the unguided chain is far from the guided one
    plain = P.Sampler(model, tree, B, S, steps=6, w=None, method=method, eta=eta)
    plain.sched.timesteps, plain.sched.alphas_cumprod = ts, SR.alphas_cumprod()[ts]
    unguided = plain.sample(nb, z_init=z0.numpy(), noises=[x.numpy() for x in noises])
    assert rel_l2(out, ref) < 2e-3
    assert rel_l2(unguided, ref) > 1e-2


# ---- 4. graph replay and eager ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
def test_graph_replay_and_eager_are_bit_identical(dtype):
    S, B = 16, 2
    model, _, _, tree, batch, _ = _setup(TINY64, S, B, dtype, params='random')
    nb = np_batch(batch)
    views, poses, K, targets = _two_view_pool(B, S)
    guide = P.XUNet(**TINY, dtype=dtype)
    gparams = _random_params(TINY, S, 8)
    out = {}
    for use_graph in (True, False):
        res = []
        for kw in (dict(method='ddpm'), dict(method='dpmpp_2m', dynamic_threshold=0.9, cache_interval=2, cache_level=1)):
            samp = P.Sampler(model, tree, B, S, steps=8, w=2.0, use_graph=use_graph, guide_params=gparams,
                             guide_model=guide, **kw)
            res += [samp.sample(nb, seed=3), samp.sample_views(views, poses, K, targets, seed=3)]
        out[use_graph] = res
    for a, b in zip(out[True], out[False]):
        assert bool(torch.isfinite(a).all())
        assert torch.equal(a, b)


# ---- 5. the samplers without a guide are untouched ------------------------------------------------------------------------
def test_unguided_samplers_unchanged_after_an_autoguided_run():
    S, B = 64, 2
    model, _, _, tree, batch, _ = _setup(SMALL, S, B, 'bf16', params='random')
    nb = np_batch(batch)
    plain = [P.Sampler(model, tree, B, S, steps=6, w=None, method='dpmpp_2m'), P.Sampler(model, tree, B, S, steps=6, w=3.0)]
    before = [s.sample(nb, seed=2) for s in plain]
    P.Sampler(model, tree, B, S, steps=6, w=2.0, method='dpmpp_2m', guide_params=_random_params(SMALL, S, 8),
              cache_interval=2, cache_level=1).sample(nb, seed=2)
    after = [s.sample(nb, seed=2) for s in plain]
    fresh = [P.Sampler(model, tree, B, S, steps=6, w=None, method='dpmpp_2m').sample(nb, seed=2),
             P.Sampler(model, tree, B, S, steps=6, w=3.0).sample(nb, seed=2)]
    for a, b, c in zip(before, after, fresh):
        assert torch.equal(a, b) and torch.equal(a, c)


# ---- the step entry against the guided steps -----------------------------------------------------------------------------
@pytest.mark.parametrize('mode', ['table', 'multistep', 'dynamic', 'dynamic_multistep'])
def test_guide_step_is_the_guided_step_on_two_outputs(lib, mode):
    """xunet_sampler_step_guide(a, b, w) gives the bits of the guided entries on [a ; b] at the same w: z, x0_hist, the next
    z (B rows) and log-SNR, and the per-view scale."""
    B, S, w = 3, 16, 1.7
    n = B * S * S * 3
    method = 'dpmpp_2m' if 'multistep' in mode else 'ddim'
    rows, _ = sampler_table(Schedule(6, spacing='logsnr' if method == 'dpmpp_2m' else 'linear'), method,
                            eta=0.5 if method == 'ddim' else 0.0)
    tab = torch.tensor(rows, dtype=torch.float32, device='cuda')
    gen = torch.Generator(device='cuda').manual_seed(0)
    a, b = (torch.randn(n, generator=gen, device='cuda') * 3 for _ in range(2))
    z0 = torch.randn(n, generator=gen, device='cuda')
    seed = torch.full((1,), 77, dtype=torch.int64, device='cuda')
    p = 0.9 if 'dynamic' in mode else 0.0
    hist = 'multistep' in mode
    res = {}
    for entry in ('guided', 'guide'):
        z = z0.clone()
        pos = torch.zeros(1, dtype=torch.int32, device='cuda')
        x0h = torch.zeros(n, device='cuda') if hist else None
        scale = torch.zeros(B, device='cuda')
        nz, nl = torch.zeros(2 * n, device='cuda'), torch.zeros(2 * B, device='cuda')
        hp = None if x0h is None else x0h.data_ptr()
        for _ in range(3):
            if entry == 'guide':
                rc = lib.xunet_sampler_step_guide(a.data_ptr(), b.data_ptr(), z.data_ptr(), None, n, w, tab.data_ptr(),
                                                  pos.data_ptr(), seed.data_ptr(), hp, B, p,
                                                  scale.data_ptr() if p else None, nz.data_ptr(), nl.data_ptr(), _stream())
            else:
                e2 = torch.cat([a, b])
                head = (e2.data_ptr(), z.data_ptr(), None, n, w, tab.data_ptr(), pos.data_ptr(), seed.data_ptr())
                tail = (nz.data_ptr(), nl.data_ptr(), 2 * B, _stream())
                if p:
                    rc = lib.xunet_sampler_step_dynamic(*head, hp, B, p, scale.data_ptr(), *tail)
                elif hist:
                    rc = lib.xunet_sampler_step_multistep(*head, hp, *tail)
                else:
                    rc = lib.xunet_sampler_step_table(*head, *tail)
            assert rc == 0, lib.xunet_last_error()
            pos.add_(1)
        torch.cuda.synchronize()
        res[entry] = (z, x0h, nz, nl, scale)
    zg, hg, nzg, nlg, sg = res['guide']
    zr, hr, nzr, nlr, sr = res['guided']
    assert torch.equal(zg, zr) and bool(torch.isfinite(zg).all())
    assert hg is None or torch.equal(hg, hr)
    assert torch.equal(nzg[:n], zg) and bool((nzg[n:] == 0).all())        # B rows only
    assert torch.equal(nlg[:B], nlr[:B]) and bool((nlg[B:] == 0).all())
    assert torch.equal(sg, sr)
    if p:
        assert bool((sg > 1).any())


# ---- 6. argument errors ----------------------------------------------------------------------------------------------------
def test_sampler_rejects_bad_guide_arguments():
    S, B = 16, 1
    model, _, _, tree, _, _ = _setup(TINY64, S, B, 'fp32', params='random')
    narrow = P.XUNet(**TINY, dtype='fp32')
    with pytest.raises(ValueError):
        P.Sampler(model, tree, B, S, steps=6, w=None, guide_params=tree)
    with pytest.raises(ValueError):
        P.Sampler(model, tree, B, S, steps=6, w=1.0, guide_model=narrow)
    # the guide tree must match the guide config: a nested dict and a flat-backed tree of the wrong width
    with pytest.raises(ValueError):
        P.Sampler(model, tree, B, S, steps=6, w=1.0, guide_params=_random_params(TINY64, S, 8), guide_model=narrow)
    with pytest.raises(ValueError):
        P.Sampler(model, tree, B, S, steps=6, w=1.0, guide_params=tree, guide_model=narrow)
    with pytest.raises(ValueError):
        P.Sampler(model, tree, B, S, steps=6, w=1.0, guide_params={'Dense_0': {}}, guide_model=narrow)
    # a cache level the guide does not have (a 3-level model guided by a 2-level one)
    deep = P.XUNet(**THREE, dtype='fp32')
    with pytest.raises(ValueError):
        P.Sampler(deep, {}, B, 32, steps=6, w=1.0, guide_params={}, guide_model=P.XUNet(**TINY, dtype='fp32'),
                  cache_interval=2, cache_level=2)


def test_guide_entry_rejects_bad_arguments(lib):
    B, S = 2, 16
    n = B * S * S * 3
    buf = [torch.zeros(n, device='cuda') for _ in range(4)]
    tab = torch.zeros(8, device='cuda')
    pos = torch.zeros(1, dtype=torch.int32, device='cuda')
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    nl = torch.zeros(B, device='cuda')
    ok = dict(out_main=buf[0].data_ptr(), out_guide=buf[1].data_ptr(), z=buf[2].data_ptr(), n=n, table=tab.data_ptr(),
              pos=pos.data_ptr(), seed=seed.data_ptr(), batch=B, percentile=0.0, next_z=buf[3].data_ptr(),
              next_logsnr=nl.data_ptr())

    def call(**kw):
        a = dict(ok, **kw)
        return lib.xunet_sampler_step_guide(a['out_main'], a['out_guide'], a['z'], None, a['n'], 1.0, a['table'], a['pos'],
                                            a['seed'], None, a['batch'], a['percentile'], None, a['next_z'],
                                            a['next_logsnr'], _stream())

    assert call() == 0, lib.xunet_last_error()
    for key in ('out_main', 'out_guide', 'z', 'table', 'pos', 'seed', 'next_z', 'next_logsnr'):
        assert call(**{key: None}) != 0, key
        assert b'xunet_sampler_step_guide' in lib.xunet_last_error()
    for bad in (dict(n=0), dict(n=-n), dict(batch=0), dict(batch=-1), dict(n=n - 1), dict(percentile=-0.5),
                dict(percentile=1.5), dict(percentile=math.nan), dict(n=2 * 256 * 256 * 3 + 6, batch=2, percentile=0.5)):
        assert call(**bad) != 0, bad
        assert b'xunet_sampler_step_guide' in lib.xunet_last_error()
    torch.cuda.synchronize()
