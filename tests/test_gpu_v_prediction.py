"""v-prediction on the GPU: xunet_forward_diffusion_v and xunet_srn_batch_v bit for bit against numpy and their eps
counterparts, a v TrainStep(data=..) against the same step fed the restated v target, the loss and gradient against an
autograd MSE on v, the sampler step kernels reading v, the Sampler under CUDA graphs, and a short training run."""
import ctypes as C

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip('cv2')
import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import srn_data as D
from novel_view_synthesis_3d_b200.diffusion import diffusion_tables, min_snr_weights, v_target
from novel_view_synthesis_3d_b200.sampling import Schedule, logsnr_schedule_cosine, sampler_table
from novel_view_synthesis_3d_b200.synthetic import synthetic_batch
from novel_view_synthesis_3d_b200.xunet import InputSlots
from tests import solver_ref as SR
from tests.device_data_ref import M64, mix64
from tests.test_gpu_device_data import CFG, _write_tree
from tests.test_gpu_model import _pool_from_batch, _setup
from tests.util import np_batch, rel_l2

pytestmark = pytest.mark.gpu

TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.0)


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return _write_tree(tmp_path_factory.mktemp('srn_v'))


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a


def _tables():
    return tuple(torch.as_tensor(a).cuda() for a in diffusion_tables())


def _nan(n, offset=0):
    """n fp32 NaNs on the device, starting `offset` floats into the allocation (offset 1: not 16-byte aligned)."""
    return torch.full((n + offset,), float('nan'), device='cuda')[offset:]


# ---- 1. xunet_forward_diffusion_v ----------------------------------------------------------------------------------------------
def _fd(lib, x0, seed, B, per, *, v, noise_in=None, t_in=None, keep_noise=True, p_uncond=0.3):
    sa, sb = _tables()
    z, noise, vv = _nan(B * per), _nan(B * per), _nan(B * per)
    logsnr, cm = _nan(B), _nan(B)
    t = torch.full((B,), -1, dtype=torch.int32, device='cuda')
    ptr = lambda a: None if a is None else a.data_ptr()
    head = (x0.data_ptr(), ptr(noise_in), ptr(t_in), seed, sa.data_ptr(), sb.data_ptr(), p_uncond, z.data_ptr())
    tail = (logsnr.data_ptr(), None if t_in is not None else t.data_ptr(), cm.data_ptr(), B, per, _stream())
    if v:
        rc = lib.xunet_forward_diffusion_v(*head, noise.data_ptr() if keep_noise else None, vv.data_ptr(), *tail)
    else:
        rc = lib.xunet_forward_diffusion(*head, noise.data_ptr(), *tail)
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    if t_in is not None:
        t = t_in
    return dict(z=z, noise=noise, v=vv, logsnr=logsnr, cond_mask=cm, t=t)


def _z_np(x0, noise, t):
    """z as the kernels contract it: fma(sqrt_ac[t], x0, fl32(sqrt_1mac[t] noise)), the fma in extended precision."""
    sa, sb = diffusion_tables()
    shape = (len(t),) + (1,) * (x0.ndim - 1)
    a, r = sa[t].reshape(shape), (sb[t].reshape(shape) * noise).astype(np.float32)
    return (a.astype(np.longdouble) * x0.astype(np.longdouble) + r.astype(np.longdouble)).astype(np.float32)


def _draws_np(seed, B, p_uncond):
    """t and cond_mask of xu_fd_sample_hash / xu_fd_timestep / xu_fd_cond_mask (common.cuh)."""
    hb = [mix64((seed * 0x9E3779B97F4A7C15 + 0xABCDEF0123 + b) & M64) for b in range(B)]
    t = np.array([h % 1000 for h in hb], np.int32)
    u = np.array([np.float32(mix64((h + 0x51ED27) & M64) >> 40) * np.float32(1.0 / 16777216.0) for h in hb], np.float32)
    return t, (u > np.float32(p_uncond)).astype(np.float32)


def test_forward_diffusion_v_matches_numpy_and_the_eps_entry(lib):
    B, S = 6, 16
    per = S * S * 3
    rng = np.random.RandomState(0)
    x0_np = rng.uniform(-1, 1, (B, S, S, 3)).astype(np.float32)
    x0 = torch.from_numpy(x0_np).cuda()
    seed = 0x1234567890ABCDEF
    eps = _fd(lib, x0, seed, B, per, v=False)
    for keep in (True, False):
        got = _fd(lib, x0, seed, B, per, v=True, keep_noise=keep)
        for key in ('z', 'logsnr', 'cond_mask', 't'):
            assert np.array_equal(_bits(got[key]), _bits(eps[key])), key
        if keep:
            assert np.array_equal(_bits(got['noise']), _bits(eps['noise']))
        else:
            assert bool(torch.isnan(got['noise']).all())                   # not written
        t = eps['t'].cpu().numpy()
        want = v_target(x0_np, eps['noise'].cpu().numpy().reshape(B, S, S, 3), t)
        assert np.array_equal(_bits(got['v']).reshape(B, -1), want.reshape(B, -1).view(np.int32))
    t_np, cm_np = _draws_np(seed, B, 0.3)
    assert np.array_equal(eps['t'].cpu().numpy(), t_np) and np.array_equal(_bits(eps['cond_mask']), _bits(cm_np))
    # fixed noise and timesteps (including both ends of the schedule): every output against numpy
    noise_np = rng.randn(B, S, S, 3).astype(np.float32)
    t_fix = np.array([0, 1, 500, 990, 998, 999], np.int32)
    got = _fd(lib, x0, seed, B, per, v=True, noise_in=torch.from_numpy(noise_np).cuda(),
              t_in=torch.from_numpy(t_fix).cuda(), keep_noise=False)
    assert np.array_equal(_bits(got['v']), v_target(x0_np, noise_np, t_fix).reshape(-1).view(np.int32))
    assert np.array_equal(_bits(got['z']), _z_np(x0_np, noise_np, t_fix).reshape(-1).view(np.int32))
    # the device's libm in double, rounded to fp32: within an ulp of numpy's (the value at t = 500 is 0 up to rounding)
    np.testing.assert_allclose(got['logsnr'].cpu().numpy(), logsnr_schedule_cosine(t_fix / 1000.0), rtol=2 ** -23, atol=1e-12)
    assert np.array_equal(_bits(got['cond_mask']), _bits(cm_np))
    # the ForwardDiffusion wrapper puts v where the loss reads its target, with the v min-SNR weights
    eng = P.XUNet(**TINY).engine(B, S, True)
    fd = P.ForwardDiffusion(eng, p_uncond=0.3, min_snr_gamma=5.0, prediction='v')
    fd.sample(x0_np, seed, t=t_fix, noise=noise_np)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(eng.inp['noise']), _bits(got['v']).reshape(B, S, S, 3))
    assert np.array_equal(_bits(eng.inp['z']), _bits(got['z']).reshape(B, S, S, 3))
    assert np.array_equal(_bits(fd.loss_weight), min_snr_weights(5.0, prediction='v').astype(np.float32)[t_fix].view(np.int32))
    # a NULL v_out is refused
    sa, sb = _tables()
    assert lib.xunet_forward_diffusion_v(x0.data_ptr(), None, None, 1, sa.data_ptr(), sb.data_ptr(), 0.1,
                                         got['z'].data_ptr(), None, None, got['logsnr'].data_ptr(), None, None, B, per,
                                         _stream()) != 0


# ---- 2. xunet_srn_batch_v --------------------------------------------------------------------------------------------------------
def _srn(lib, store, slots, count, j, k, rank, world, seed, *, v, offset, keep_noise=True, gamma=None):
    """One batch launch into slot 0 of `slots`, the noise / v buffers `offset` floats off 16-byte alignment."""
    B, S = slots.B, store.S
    n = B * S * S * 3
    step_dev = torch.full((1,), count + 1, dtype=torch.int64, device='cuda')
    idx = torch.full((B, 3), -1, dtype=torch.int32, device='cuda')
    t = torch.full((B,), -1, dtype=torch.int32, device='cuda')
    noise, vv = _nan(n, offset), _nan(n, offset)
    sa, sb = _tables()
    w = None if gamma is None else torch.as_tensor(min_snr_weights(gamma, prediction='v'), dtype=torch.float32).cuda()
    head = (C.byref(store.c_store), step_dev.data_ptr(), seed, j, k, rank, world, B, sa.data_ptr(), sb.data_ptr(), 0.1,
            None if w is None else w.data_ptr(), C.byref(slots.cbatch[0]))
    tail = (slots.inp[0]['loss_weight'].data_ptr(), idx.data_ptr(), t.data_ptr(), _stream())
    if v:
        rc = lib.xunet_srn_batch_v(*head, noise.data_ptr() if keep_noise else None, vv.data_ptr(), *tail)
    else:
        rc = lib.xunet_srn_batch(*head, noise.data_ptr(), *tail)
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    out = {key: slots.inp[0][key].clone() for key in ('x', 'z', 'logsnr', 'R1', 't1', 'R2', 't2', 'K', 'cond_mask',
                                                       'loss_weight')}
    return dict(out, noise=noise, v=vv, idx=idx.cpu().numpy().astype(np.int64), t=t.cpu().numpy())


def _targets(ds, idx, S):
    return np.stack([D.load_rgb(ds.instances[i]['imgs'][v2], S) for i, _, v2 in idx])


@pytest.mark.parametrize('S,storage,offset', [(32, 'uint8', 0), (16, 'float32', 0), (16, 'float32', 1)])
def test_srn_batch_v_matches_numpy_and_the_eps_entry(tree, lib, S, storage, offset):
    """offset 1 puts the noise / v buffers off 16-byte alignment: the kernels' scalar path."""
    store = D.DeviceScenes(tree, S)
    assert store.storage == storage
    ds = D.SRNScenes(tree, img_sidelength=S)
    B, seed = 5, 0x5EED
    slots = InputSlots(B, S, 1, store.device)
    for count, j, k, rank, world in ((0, 0, 1, 0, 1), (3, 1, 2, 0, 1), (7, 2, 3, 3, 4)):
        eps = _srn(lib, store, slots, count, j, k, rank, world, seed, v=False, offset=offset, gamma=5.0)
        for keep in (True, False):
            got = _srn(lib, store, slots, count, j, k, rank, world, seed, v=True, offset=offset, keep_noise=keep, gamma=5.0)
            for key in ('x', 'z', 'logsnr', 'R1', 't1', 'R2', 't2', 'K', 'cond_mask', 'loss_weight', 'idx', 't'):
                assert np.array_equal(_bits(got[key]), _bits(eps[key])), key
            if keep:
                assert np.array_equal(_bits(got['noise']), _bits(eps['noise']))
            else:
                assert bool(torch.isnan(got['noise']).all())
            x0 = _targets(ds, eps['idx'], S)
            want = v_target(x0, eps['noise'].cpu().numpy().reshape(B, S, S, 3), eps['t'])
            assert np.array_equal(_bits(got['v']), want.reshape(-1).view(np.int32))
        assert np.array_equal(_bits(eps['loss_weight']), min_snr_weights(5.0, prediction='v').astype(np.float32)[eps['t']].view(np.int32))
        if offset == 0:
            noise = eps['noise'].cpu().numpy().reshape(B, S, S, 3)
            assert np.array_equal(_bits(eps['z']), _z_np(x0, noise, eps['t']).view(np.int32))
    # a NULL v_out is refused
    sa, sb = _tables()
    step_dev = torch.ones(1, dtype=torch.int64, device='cuda')
    assert lib.xunet_srn_batch_v(C.byref(store.c_store), step_dev.data_ptr(), seed, 0, 1, 0, 1, B, sa.data_ptr(),
                                 sb.data_ptr(), 0.1, None, C.byref(slots.cbatch[0]), slots.inp[0]['noise'].data_ptr(), None,
                                 None, None, None, _stream()) != 0


# ---- 3. a v training step from the store equals the host-input step on the restated v target ----------------------------------
def _vstate(B=4, S=16, model_cfg=CFG, **kw):
    return P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(**model_cfg), zero_init=False, loss='mse', prediction='v',
                                **kw)


@pytest.mark.parametrize('gamma,k', [(5.0, 1), (None, 2)])
def test_v_training_from_the_store_equals_training_on_the_restated_targets(tree, lib, gamma, k):
    S, B, seed = 16, 4, 9
    store = D.DeviceScenes(tree, S)
    ds = D.SRNScenes(tree, img_sidelength=S)
    sa, sb = _vstate(), _vstate()
    assert sa.prediction == 'v'
    step_a = P.TrainStep(sa, data=store, data_seed=seed, grad_accum_steps=k, min_snr_gamma=gamma)
    step_b = P.TrainStep(sb, grad_accum_steps=k)
    slots = InputSlots(B, S, 1, store.device)
    for c in range(3):
        parts = []
        for j in range(k):
            got = _srn(lib, store, slots, c, j, k, 0, 1, seed, v=False, offset=0, gamma=gamma)
            noise = got['noise'].cpu().numpy().reshape(B, S, S, 3)
            got['target'] = torch.from_numpy(v_target(_targets(ds, got['idx'], S), noise, got['t'])).cuda()
            parts.append(got)
        cat = lambda key: torch.cat([p[key] for p in parts]).clone()
        batch = {key: cat(key) for key in ('x', 'z', 'logsnr', 'R1', 't1', 'R2', 't2', 'K')}
        la = float(step_a())
        lb = float(step_b(batch, cat('target'), cond_mask=cat('cond_mask'), loss_weight=cat('loss_weight')))
        torch.cuda.synchronize()
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32), (c, la, lb)
        assert torch.equal(step_a.eng.grads.view(torch.int32), step_b.eng.grads.view(torch.int32)), c
    for x, y in ((sa.params.flat, sb.params.flat), (sa.opt_state.mu, sb.opt_state.mu), (sa.opt_state.nu, sb.opt_state.nu)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert step_a.h2d_bytes == 0


def test_v_loss_and_gradient_equal_an_autograd_mse_on_v():
    S, B = 16, 3
    model = P.XUNet(**TINY, dtype='fp32')
    st = P.create_train_state(0, 1, 1e-4, B, S, model=model, zero_init=False, loss='mse', prediction='v')
    batch, _ = synthetic_batch(B, S, seed=4)
    rng = np.random.RandomState(5)
    x0 = rng.uniform(-1, 1, (B, S, S, 3)).astype(np.float32)
    noise = rng.randn(B, S, S, 3).astype(np.float32)
    t = np.array([3, 500, 999])
    sqa, sqb = diffusion_tables()
    batch = dict(batch, z=(sqa[t][:, None, None, None] * x0 + sqb[t][:, None, None, None] * noise).astype(np.float32),
                 logsnr=logsnr_schedule_cosine(t / 1000.0))
    nb = {key: np.asarray(val, np.float32) for key, val in batch.items()}
    v = v_target(x0, noise, t)
    cond = np.array([1.0, 0.0, 1.0], np.float32)
    loss, grads = P.apply_model(st, nb['x'], nb['z'], nb['logsnr'], nb['R1'], nb['t1'], nb['R2'], nb['t2'], nb['K'], v,
                                cond_mask=cond)
    loss, g = float(loss), grads.flat.clone()
    flat = st.params.flat.detach().clone().requires_grad_(True)
    out = model.apply_autograd(flat, nb, cond_mask=cond, train=True)
    ref = (out - torch.from_numpy(v).cuda()).pow(2).mean()
    ref.backward()
    torch.cuda.synchronize()
    assert loss == pytest.approx(float(ref.detach()), rel=1e-6)
    assert bool((g != 0).any())
    assert rel_l2(g, flat.grad) < 1e-5, rel_l2(g, flat.grad)


# ---- 4. the step kernels read v ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('method,eta,spacing,dynamic', [('ddpm', 0.0, 'linear', False), ('ddim', 0.5, 'linear', False),
                                                        ('dpmpp_2m', 0.0, 'logsnr', False), ('ddim', 0.0, 'linear', True),
                                                        ('dpmpp_2m', 0.0, 'logsnr', True)])
def test_step_kernels_fed_the_v_of_a_known_x0_take_the_fp64_step(lib, method, eta, spacing, dynamic):
    """Every step gets out2 = [v; v], v the exact v of a fixed x0 at the current z, and guidance w = 3: the kernel's z' is the
    fp64 update from that x0 at fp32 tolerance, from t = 999 down to 0."""
    sched = Schedule(10, spacing=spacing)
    rows, _ = sampler_table(sched, method, eta=eta, prediction='v')
    ac = SR.alphas_cumprod()
    ts = list(sched.timesteps[::-1])
    assert ts[0] == 999 and ts[-1] == 0
    B, per = 2, 8 * 8 * 3
    n = B * per
    g = torch.Generator().manual_seed(11)
    x0 = torch.rand(n, generator=g, dtype=torch.float64) * 1.8 - 0.9
    noise = torch.randn(len(ts), n, generator=g, dtype=torch.float64)
    tab, nd = torch.tensor(rows).float().cuda(), noise.float().cuda()
    z = torch.randn(n, generator=g, dtype=torch.float64).float().cuda()
    pos = torch.zeros(1, dtype=torch.int32, device='cuda')
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    hist = torch.full((n,), float('nan'), device='cuda') if method == 'dpmpp_2m' else None
    scale = torch.zeros(B, device='cuda')
    next_z2, next_logsnr2 = torch.zeros(2 * n, device='cuda'), torch.zeros(2 * B, device='cuda')
    for k, t in enumerate(ts):
        zc = z.double().cpu()
        a = ac[t]
        v = (np.sqrt(a) * zc - x0) / np.sqrt(1. - a)                  # x0 = sqrt(a) z - sqrt(1 - a) v
        out2 = torch.cat([v, v]).float().cuda()
        r = rows[k]
        ref = r[2] * x0 + r[3] * zc + r[4] * noise[k] + (r[6] * x0 if r[6] != 0 else 0.)
        head = (out2.data_ptr(), z.data_ptr(), nd.data_ptr(), n, 3.0, tab.data_ptr(), pos.data_ptr(), seed.data_ptr())
        tail = (next_z2.data_ptr(), next_logsnr2.data_ptr(), 2 * B, _stream())
        if dynamic:
            rc = lib.xunet_sampler_step_dynamic(*head, None if hist is None else hist.data_ptr(), B, 0.995, scale.data_ptr(),
                                                *tail)
        elif hist is None:
            rc = lib.xunet_sampler_step_table(*head, *tail)
        else:
            rc = lib.xunet_sampler_step_multistep(*head, hist.data_ptr(), *tail)
        assert rc == 0, lib.xunet_last_error()
        pos.add_(1)
        torch.cuda.synchronize()
        err = float((z.double().cpu() - ref).abs().max())
        assert err <= 2e-5 * max(1.0, float(ref.abs().max())), (k, t, err)
        if hist is not None:
            assert float((hist.double().cpu() - x0).abs().max()) <= 2e-5, (k, t)
        if dynamic:
            assert bool((scale == 1.0).all())                             # |x0| <= 0.9: the fixed clip's bits
    assert float((z.double().cpu() - x0).abs().max()) <= 2e-5               # the last step returns x0


# ---- 5. the Sampler with prediction='v' ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('method,eta,dynamic', [('ddpm', 0.0, None), ('ddim', 0.5, None), ('dpmpp_2m', 0.0, None),
                                                ('ddim', 0.0, 0.995)])
def test_v_sampler_graph_replay_equals_eager(method, eta, dynamic):
    S_, B = 16, 2
    model, _, _, tree_, batch, _ = _setup(TINY, S_, B, 'bf16')
    nb = np_batch(batch)
    views, poses, K, tp = _pool_from_batch(nb)
    tp = {key: np.concatenate([tp[key], poses[key]], 1) for key in ('R', 't')}
    out = {}
    for use_graph in (True, False):
        samp = P.Sampler(model, tree_, B, S_, steps=8, w=3.0, use_graph=use_graph, method=method, eta=eta,
                         dynamic_threshold=dynamic, prediction='v')
        assert samp.prediction == 'v' and not samp.logsnr_lag
        out[use_graph] = (samp.sample(nb, seed=3), samp.sample_views(views, poses, K, tp, seed=3))
        rows, first = sampler_table(samp.sched, method, eta=eta, logsnr_lag=False, prediction='v')
        assert torch.equal(samp._tab.cpu(), torch.as_tensor(rows, dtype=torch.float32))
    assert torch.equal(out[True][0], out[False][0]) and torch.equal(out[True][1], out[False][1])
    assert bool(torch.isfinite(out[True][0]).all()) and bool(torch.isfinite(out[True][1]).all())
    # the same network read as eps samples something else
    eps = P.Sampler(model, tree_, B, S_, steps=8, w=3.0, method=method, eta=eta, dynamic_threshold=dynamic,
                    logsnr_lag=False).sample(nb, seed=3)
    assert not torch.equal(eps, out[True][0])


def test_v_sampler_arguments():
    model, _, _, tree_, _, _ = _setup(TINY, 16, 1, 'fp32')
    with pytest.raises(ValueError):
        P.Sampler(model, tree_, 1, 16, steps=6, prediction='x0')
    assert P.Sampler(model, tree_, 1, 16, steps=6).logsnr_lag                          # the eps default is unchanged
    assert P.Sampler(model, tree_, 1, 16, steps=6, prediction='v', logsnr_lag=True).logsnr_lag


# ---- 6. a short v training run learns -----------------------------------------------------------------------------------------
def test_short_v_training_run_lowers_the_loss(tree):
    store = D.DeviceScenes(tree, 16)
    st = _vstate(B=4, S=16, model_cfg=dict(CFG, dropout=0.0))
    step = P.TrainStep(st, data=store, data_seed=1, min_snr_gamma=5.0)
    losses = [float(step()) for _ in range(120)]
    assert np.isfinite(losses).all()
    first, last = np.mean(losses[:20]), np.mean(losses[-20:])
    assert last < 0.9 * first, (first, last)
