"""Progressive distillation on the GPU: xunet_srn_batch_distill against numpy and xunet_srn_batch_v, the teacher step against
xunet_sampler_step_table, the target kernel against an fp32 numpy restatement, the three kernels and the student's DDIM
grid together, the captured distillation TrainStep against an eager composition, the unguided sampler step against the
guided one at w = 0, Sampler(w=None) under CUDA graphs, and a short distillation run."""
import ctypes as C

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip('cv2')
import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200 import srn_data as D
from novel_view_synthesis_3d_b200.diffusion import diffusion_tables
from novel_view_synthesis_3d_b200.distill import Teacher, create_distill_state, target_table
from novel_view_synthesis_3d_b200.sampling import Schedule, distill_grid, logsnr_schedule_cosine, sampler_table
from novel_view_synthesis_3d_b200.xunet import InputSlots
from tests import solver_ref as SR
from tests.device_data_ref import M64, mix64
from tests.test_gpu_device_data import CFG, _write_tree
from tests.test_gpu_model import _pool_from_batch, _setup
from tests.test_gpu_v_prediction import TINY, _bits, _nan, _srn, _stream, _tables, _targets, _z_np
from tests.util import np_batch

pytestmark = pytest.mark.gpu

BATCH_KEYS = ('x', 'z', 'logsnr', 'R1', 't1', 'R2', 't2', 'K')


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return _write_tree(tmp_path_factory.mktemp('srn_distill'))


def _ld(a):
    return np.asarray(a, np.float32).astype(np.longdouble)


def _fma(a, b, c):
    """fp32 fma: the exact product plus c in extended precision, rounded to fp32."""
    return (_ld(a) * _ld(b) + _ld(c)).astype(np.float32)


def _teacher_rows(B, S, copies, offset=0):
    """Teacher input rows in fresh NaN buffers (offset 1: off 16-byte alignment) and their xunet_batch."""
    n = copies * B * S * S * 3
    bufs = {'x': _nan(n, offset), 'z': _nan(n, offset), 'logsnr': _nan(copies * B), 'R1': _nan(copies * B * 9),
            't1': _nan(copies * B * 3), 'R2': _nan(copies * B * 9), 't2': _nan(copies * B * 3), 'K': _nan(copies * B * 9),
            'cond_mask': _nan(copies * B)}
    cb = _lib.XunetBatch(**{k: v.data_ptr() for k, v in bufs.items()}, rays=None)
    return bufs, cb


def _distill_draw(lib, store, slots, cb, copies, count, j, k, rank, world, seed, grid):
    B = slots.B
    step_dev = torch.full((1,), count + 1, dtype=torch.int64, device='cuda')
    g = torch.as_tensor(np.asarray(grid), dtype=torch.int32, device='cuda')
    m = torch.full((B,), -1, dtype=torch.int32, device='cuda')
    idx = torch.full((B, 3), -1, dtype=torch.int32, device='cuda')
    t = torch.full((B,), -1, dtype=torch.int32, device='cuda')
    sa, sb = _tables()
    slots.inp[0]['noise'].fill_(float('nan'))
    rc = lib.xunet_srn_batch_distill(C.byref(store.c_store), step_dev.data_ptr(), seed, j, k, rank, world, B, sa.data_ptr(),
                                     sb.data_ptr(), g.data_ptr(), len(grid), C.byref(slots.cbatch[0]), C.byref(cb), copies,
                                     m.data_ptr(), idx.data_ptr(), t.data_ptr(), _stream())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    out = {key: slots.inp[0][key].clone() for key in BATCH_KEYS + ('cond_mask', 'noise')}
    return dict(out, m=m.cpu().numpy(), idx=idx.cpu().numpy().astype(np.int64), t=t.cpu().numpy())


# ---- 1. the distillation batch draw -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('S,storage,offset', [(32, 'uint8', 0), (16, 'float32', 0), (16, 'float32', 1)])
def test_distill_batch_matches_numpy_and_the_v_draw(tree, lib, S, storage, offset):
    """offset 1 puts the teacher rows off 16-byte alignment: the kernel's scalar path."""
    store = D.DeviceScenes(tree, S)
    assert store.storage == storage
    ds = D.SRNScenes(tree, img_sidelength=S)
    B, seed = 5, 0x5EED
    per = S * S * 3
    slots, vslots = InputSlots(B, S, 1, store.device), InputSlots(B, S, 1, store.device)
    sa_np, sb_np = diffusion_tables()
    for copies in (2, 1):
        for count, j, k, rank, world in ((0, 0, 1, 0, 1), (3, 1, 2, 0, 1), (7, 2, 3, 3, 4)):
            ref = _srn(lib, store, vslots, count, j, k, rank, world, seed, v=True, offset=offset)
            rows, cb = _teacher_rows(B, S, copies, offset)
            # grid = 0..999 in order: m = t of the plain draw, so every student row equals xunet_srn_batch_v's
            got = _distill_draw(lib, store, slots, cb, copies, count, j, k, rank, world, seed, np.arange(1000))
            for key in BATCH_KEYS + ('idx', 't'):
                assert np.array_equal(_bits(got[key]), _bits(ref[key])), key
            assert np.array_equal(got['m'], ref['t']) and bool((got['cond_mask'] == 1).all())
            assert bool(torch.isnan(got['noise']).all())                      # no target is written
            # a distillation grid: t = grid[hash mod N], z and logsnr follow it
            grid = distill_grid(64, 1)
            got = _distill_draw(lib, store, slots, cb, copies, count, j, k, rank, world, seed, grid)
            s = D.diffusion_seed(seed, count, j, k, rank)
            hb = [mix64((s * 0x9E3779B97F4A7C15 + 0xABCDEF0123 + b) & M64) for b in range(B)]
            m_np = np.array([h % len(grid) for h in hb])
            assert np.array_equal(got['m'], m_np) and np.array_equal(got['t'], grid[m_np])
            for key in ('x', 'R1', 't1', 'R2', 't2', 'K', 'idx'):
                assert np.array_equal(_bits(got[key]), _bits(ref[key])), key
            x0 = _targets(ds, got['idx'], S)
            noise = ref['noise'].cpu().numpy().reshape(B, S, S, 3)
            t = got['t']
            if offset == 0:
                want = _z_np(x0, noise, t)
            else:     # the scalar path contracts the other product: fma(sqrt_1mac, noise, fl(sqrt_ac x0))
                shp = (B, 1, 1, 1)
                want = _fma(sb_np[t].reshape(shp), noise, (sa_np[t].reshape(shp) * x0).astype(np.float32))
            assert np.array_equal(_bits(got['z']), want.view(np.int32))
            np.testing.assert_allclose(got['logsnr'].cpu().numpy(), logsnr_schedule_cosine(t / 1000.0), rtol=2 ** -23,
                                       atol=1e-12)
            for c in range(copies):
                for key in BATCH_KEYS:
                    n = got[key][0].numel()
                    trow = rows[key][c * B * n:(c + 1) * B * n]
                    assert np.array_equal(_bits(trow), _bits(got[key]).reshape(-1)), (c, key)
            assert bool(torch.isnan(rows['cond_mask']).all())                  # set once by the caller, never here
    # bad arguments are refused
    rows, cb = _teacher_rows(B, S, 2)
    sa, sb = _tables()
    g = torch.arange(10, dtype=torch.int32, device='cuda')
    m = torch.zeros(B, dtype=torch.int32, device='cuda')
    step_dev = torch.ones(1, dtype=torch.int64, device='cuda')
    call = lambda **kw: lib.xunet_srn_batch_distill(
        C.byref(store.c_store), step_dev.data_ptr(), seed, 0, 1, 0, 1, B, sa.data_ptr(), sb.data_ptr(),
        kw.get('grid', g.data_ptr()), kw.get('n_grid', 10), C.byref(slots.cbatch[0]), C.byref(cb), kw.get('copies', 2),
        kw.get('m', m.data_ptr()), None, None, _stream())
    assert call() == 0
    for kw in (dict(grid=None), dict(n_grid=0), dict(copies=3), dict(m=None)):
        assert call(**kw) != 0, kw
    torch.cuda.synchronize()


# ---- 2. the teacher step is the sampler step at pos = 2m ------------------------------------------------------------------------
def _step_table(rows):
    return torch.as_tensor(rows, dtype=torch.float32, device='cuda')


@pytest.mark.parametrize('copies,pred', [(2, 'eps'), (1, 'v'), (2, 'v')])
def test_teacher_step_is_the_sampler_step_at_2m(lib, copies, pred):
    B, S, w = 6, 8, 2.5
    per = S * S * 3
    n = B * per
    grid = distill_grid(32, 0)
    tab = _step_table(sampler_table(Schedule(timesteps=grid), 'ddim', prediction=pred, logsnr_lag=False)[0])
    g = torch.Generator(device='cuda').manual_seed(3)
    out = torch.randn(copies * n, generator=g, device='cuda') * 1.5
    z0 = torch.randn(n, generator=g, device='cuda')
    m = torch.tensor([0, 15, 7, 3, 15, 9], dtype=torch.int32, device='cuda')     # mixed, with the last interval
    rows, cb = _teacher_rows(B, S, copies)
    rows['z'][:n].copy_(z0)
    assert lib.xunet_distill_teacher_step(out.data_ptr(), w, copies, tab.data_ptr(), m.data_ptr(), B, per, C.byref(cb),
                                          _stream()) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    for b in range(B):
        sl = slice(b * per, (b + 1) * per)
        oc = out[sl]
        ou = out[n + b * per:n + (b + 1) * per] if copies == 2 else oc
        z = z0[sl].clone()
        pos = torch.full((1,), 2 * int(m[b]), dtype=torch.int32, device='cuda')
        seed = torch.zeros(1, dtype=torch.int64, device='cuda')
        nz, nl = torch.zeros(2 * per, device='cuda'), torch.zeros(2, device='cuda')
        ww = w if copies == 2 else 0.0
        assert lib.xunet_sampler_step_table(torch.cat([oc, ou]).data_ptr(), z.data_ptr(), None, per, ww, tab.data_ptr(),
                                            pos.data_ptr(), seed.data_ptr(), nz.data_ptr(), nl.data_ptr(), 2, _stream()) == 0
        torch.cuda.synchronize()
        for c in range(copies):
            assert torch.equal(rows['z'][c * n + b * per:c * n + (b + 1) * per].view(torch.int32), z.view(torch.int32)), (b, c)
            assert rows['logsnr'][c * B + b].item() == tab[2 * int(m[b]), 5].item()
    assert lib.xunet_distill_teacher_step(out.data_ptr(), w, 3, tab.data_ptr(), m.data_ptr(), B, per, C.byref(cb),
                                          _stream()) != 0


# ---- 3. the target kernel against an fp32 numpy restatement -------------------------------------------------------------------
@pytest.mark.parametrize('copies', [2, 1])
def test_target_kernel_matches_numpy(lib, copies):
    B, S, w = 5, 8, 3.0
    per = S * S * 3
    n = B * per
    grid = distill_grid(64, 1)                                   # a round-2 teacher grid: 32 rows, 16 student rows
    ttab_np = sampler_table(Schedule(timesteps=grid), 'ddim', prediction='v', logsnr_lag=False)[0].astype(np.float32)
    gtab_np = target_table(grid).astype(np.float32)
    r = np.random.RandomState(4)
    out = (r.randn(copies * n) * 0.7).astype(np.float32)
    zp = r.randn(n).astype(np.float32)
    zt = r.randn(n).astype(np.float32)
    m = np.array([0, 15, 4, 8, 15], np.int32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    v = _nan(n)
    assert lib.xunet_distill_target(dev(out).data_ptr(), w, copies, dev(ttab_np).data_ptr(), dev(gtab_np).data_ptr(),
                                    dev(m).data_ptr(), dev(zt).data_ptr(), dev(zp).data_ptr(), B, per, v.data_ptr(),
                                    _stream()) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    mb = np.repeat(m, per)
    t1, g = ttab_np[2 * mb + 1], gtab_np[mb]
    f = np.float32
    if copies == 2:
        e = _fma(f(1) + f(w), out[:n], -(f(w) * out[n:]))
    else:
        e = out[:n]
    x0 = np.clip(_fma(t1[:, 0], zp, -(t1[:, 1] * e)), f(-1), f(1))
    z2 = _fma(t1[:, 2], x0, t1[:, 3] * zp)
    xt = (g[:, 0] * z2) - (g[:, 1] * zt)
    want = ((g[:, 2] * zt) - xt) / g[:, 3]
    assert np.array_equal(_bits(v), want.astype(np.float32).view(np.int32))
    assert lib.xunet_distill_target(dev(out).data_ptr(), w, copies, dev(ttab_np).data_ptr(), None, dev(m).data_ptr(),
                                    dev(zt).data_ptr(), dev(zp).data_ptr(), B, per, v.data_ptr(), _stream()) != 0


# ---- 4. the kernels and the student grid together -------------------------------------------------------------------------------
@pytest.mark.parametrize('copies,pred', [(2, 'eps'), (1, 'v')])
def test_student_ddim_step_on_the_target_reaches_the_teachers_z2(lib, copies, pred):
    """The teacher outputs the exact prediction of a fixed x0 (|x0| <= 0.9, so no clip acts), and its second step is
    xunet_sampler_step_table at pos = 2m + 1 from the teacher step's z'.  For every student row m the unguided student step
    on its own grid, fed the v target, lands on that z'' to fp32 accuracy; z'' is alpha'' x0 + sigma'' eps (x0 after the
    last interval) up to the fp32 error of the teacher's x0."""
    B, S, w = 3, 8, 2.0
    per = S * S * 3
    n = B * per
    grid = distill_grid(32, 0)
    ttab = _step_table(sampler_table(Schedule(timesteps=grid), 'ddim', prediction=pred, logsnr_lag=False)[0])
    stab = _step_table(sampler_table(Schedule(timesteps=grid[0::2]), 'ddim', prediction='v', logsnr_lag=False)[0])
    gtab = _step_table(target_table(grid))
    ac = SR.alphas_cumprod()
    g = torch.Generator().manual_seed(5)
    x0 = torch.rand(n, generator=g, dtype=torch.float64) * 1.8 - 0.9
    eps = torch.randn(n, generator=g, dtype=torch.float64)

    def exact(z, t):
        a = ac[t]
        e = (z.double().cpu() - np.sqrt(a) * x0) / np.sqrt(1. - a)
        o = e if pred == 'eps' else np.sqrt(a) * e - np.sqrt(1. - a) * x0
        return torch.cat([o] * copies).float().cuda()
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    for mm in range(len(grid) // 2):
        t, t1 = grid[2 * mm], grid[2 * mm + 1]
        a = ac[t]
        zt = (np.sqrt(a) * x0 + np.sqrt(1. - a) * eps).float().cuda()
        m = torch.full((B,), mm, dtype=torch.int32, device='cuda')
        rows, cb = _teacher_rows(B, S, copies)
        rows['z'][:n].copy_(zt)
        assert lib.xunet_distill_teacher_step(exact(zt, t).data_ptr(), w, copies, ttab.data_ptr(), m.data_ptr(), B, per,
                                              C.byref(cb), _stream()) == 0
        v = _nan(n)
        assert lib.xunet_distill_target(exact(rows['z'][:n], t1).data_ptr(), w, copies, ttab.data_ptr(), gtab.data_ptr(),
                                        m.data_ptr(), zt.data_ptr(), rows['z'].data_ptr(), B, per, v.data_ptr(),
                                        _stream()) == 0
        out2 = exact(rows['z'][:n], t1)
        z2 = rows['z'][:n].clone()
        o2 = out2 if copies == 2 else torch.cat([out2, out2])
        pos = torch.full((1,), 2 * mm + 1, dtype=torch.int32, device='cuda')
        nz2, nl2 = torch.zeros(2 * n, device='cuda'), torch.zeros(2 * B, device='cuda')
        assert lib.xunet_sampler_step_table(o2.data_ptr(), z2.data_ptr(), None, n, w if copies == 2 else 0.0,
                                            ttab.data_ptr(), pos.data_ptr(), seed.data_ptr(), nz2.data_ptr(), nl2.data_ptr(),
                                            2 * B, _stream()) == 0
        z, nz, nl = zt.clone(), torch.zeros(n, device='cuda'), torch.zeros(B, device='cuda')
        pos = torch.full((1,), mm, dtype=torch.int32, device='cuda')
        assert lib.xunet_sampler_step_cond(v.data_ptr(), z.data_ptr(), None, n, stab.data_ptr(), pos.data_ptr(),
                                           seed.data_ptr(), None, B, 0.0, None, nz.data_ptr(), nl.data_ptr(), _stream()) == 0
        torch.cuda.synchronize()
        err = float((z - z2).abs().max())
        assert err <= 2e-5 * max(1.0, float(z2.abs().max())), (mm, t, err)
        a2 = ac[grid[2 * mm + 2]] if 2 * mm + 2 < len(grid) else 1.0
        ref = np.sqrt(a2) * x0 + np.sqrt(1. - a2) * eps
        assert float((z2.double().cpu() - ref).abs().max()) <= 2e-2, (mm, t)
        assert torch.equal(nz, z) and bool((nl == stab[mm, 5]).all())


# ---- 5. the captured distillation step equals the eager composition ---------------------------------------------------------------
def sa_eng_differs(ta, tb):
    return ta.model.engine(ta.B, ta.S, True) is not tb.model.engine(tb.B, tb.S, True) and ta.eng is not tb.eng


def _teacher_model_params(S, B, seed=0):
    model = P.XUNet(**CFG)
    st = P.create_train_state(seed, 1, 1e-3, B, S, model=model, zero_init=False)
    return model, st.params


@pytest.mark.parametrize('k,w', [(1, 2.0), (2, None)])
def test_captured_distillation_step_equals_the_eager_composition(tree, lib, k, w):
    S, B, seed = 16, 4, 21
    store = D.DeviceScenes(tree, S)
    model, params = _teacher_model_params(S, B)
    pred, rounds = ('eps', 0) if w is not None else ('v', 1)
    # two model objects: the two students must not share an engine (and so a gradient buffer)
    ta = Teacher(model, params, 32, batch_size=B, img_sidelength=S, w=w, prediction=pred, rounds=rounds)
    tb = Teacher(P.XUNet(**CFG), params, 32, batch_size=B, img_sidelength=S, w=w, prediction=pred, rounds=rounds)
    assert sa_eng_differs(ta, tb)
    sa, sb = create_distill_state(ta, 1e-3), create_distill_state(tb, 1e-3)
    assert torch.equal(sa.params.flat, ta.flat) and sa.distill == ta.record and sa.prediction == 'v' and sa.loss == 'mse'
    step_a = P.TrainStep(sa, data=store, data_seed=seed, grad_accum_steps=k, teacher=ta)
    step_b = P.TrainStep(sb, grad_accum_steps=k)
    slots = InputSlots(B, S, 1, store.device)
    per = S * S * 3
    st = _stream()
    for c in range(3):
        parts = []
        for j in range(k):
            step_dev = torch.full((1,), c + 1, dtype=torch.int64, device='cuda')
            sqa, sqb = _tables()
            assert lib.xunet_srn_batch_distill(C.byref(store.c_store), step_dev.data_ptr(), seed, j, k, 0, 1, B,
                                               sqa.data_ptr(), sqb.data_ptr(), tb.grid_t.data_ptr(), len(tb.student_grid),
                                               C.byref(slots.cbatch[0]), C.byref(tb.eng.cbatch), tb.copies, tb.m.data_ptr(),
                                               None, None, st) == 0
            tb.eng.forward(tb.flat, train=False)
            assert lib.xunet_distill_teacher_step(tb.eng.eps.data_ptr(), w or 0.0, tb.copies, tb.table.data_ptr(),
                                                  tb.m.data_ptr(), B, per, C.byref(tb.eng.cbatch), st) == 0
            tb.eng.forward(tb.flat, train=False)                          # full conditioning
            assert lib.xunet_distill_target(tb.eng.eps.data_ptr(), w or 0.0, tb.copies, tb.table.data_ptr(),
                                            tb.target.data_ptr(), tb.m.data_ptr(), slots.inp[0]['z'].data_ptr(),
                                            tb.eng.inp['z'].data_ptr(), B, per, slots.inp[0]['noise'].data_ptr(), st) == 0
            parts.append({key: slots.inp[0][key].clone() for key in BATCH_KEYS + ('cond_mask', 'noise')})
        cat = lambda key: torch.cat([p[key] for p in parts]).clone()
        batch = {key: cat(key) for key in BATCH_KEYS}
        la = float(step_a())
        lb = float(step_b(batch, cat('noise'), cond_mask=cat('cond_mask')))
        torch.cuda.synchronize()
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32), (c, la, lb)
        assert torch.equal(step_a.eng.grads.view(torch.int32), step_b.eng.grads.view(torch.int32)), c
    for x, y in ((sa.params.flat, sb.params.flat), (sa.opt_state.mu, sb.opt_state.mu), (sa.opt_state.nu, sb.opt_state.nu)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert step_a.mode == 'one_graph' and step_a.h2d_bytes == 0
    # the same step run eagerly replays the same bits
    sc = create_distill_state(tb, 1e-3)
    step_c = P.TrainStep(sc, data=store, data_seed=seed, grad_accum_steps=k, teacher=tb, use_graph=False)
    sd = create_distill_state(ta, 1e-3)
    step_d = P.TrainStep(sd, data=store, data_seed=seed, grad_accum_steps=k, teacher=ta)
    for c in range(2):
        lc, ld = float(step_c()), float(step_d())
        assert np.float32(lc).view(np.int32) == np.float32(ld).view(np.int32), c
    torch.cuda.synchronize()
    assert torch.equal(sc.params.flat.view(torch.int32), sd.params.flat.view(torch.int32))


# ---- 6. the unguided step is the guided step at w = 0 ------------------------------------------------------------------------------
@pytest.mark.parametrize('method,spacing', [('ddpm', 'linear'), ('ddim', 'linear'), ('dpmpp_2m', 'logsnr')])
@pytest.mark.parametrize('dynamic', [None, 0.9])
def test_unguided_step_equals_the_guided_step_at_w0(lib, method, spacing, dynamic):
    B, per = 3, 8 * 8 * 3
    n = B * per
    rows, _ = sampler_table(Schedule(10, spacing=spacing), method, prediction='v')
    tab = _step_table(rows)
    g = torch.Generator(device='cuda').manual_seed(7)
    z0 = torch.randn(n, generator=g, device='cuda')
    seed = torch.full((1,), 1234, dtype=torch.int64, device='cuda')
    res = {}
    for guided in (True, False):
        z = z0.clone()
        hist = torch.zeros(n, device='cuda') if method == 'dpmpp_2m' else None
        nz = torch.zeros((2 if guided else 1) * n, device='cuda')
        nl = torch.zeros((2 if guided else 1) * B, device='cuda')
        scale = torch.zeros(B, device='cuda')
        pos = torch.zeros(1, dtype=torch.int32, device='cuda')
        outs = []
        for k in range(len(rows)):
            out = torch.randn(n, generator=torch.Generator(device='cuda').manual_seed(100 + k), device='cuda') * 2
            hp = None if hist is None else hist.data_ptr()
            if guided:
                o2 = torch.cat([out, out])
                head = (o2.data_ptr(), z.data_ptr(), None, n, 0.0, tab.data_ptr(), pos.data_ptr(), seed.data_ptr())
                tail = (nz.data_ptr(), nl.data_ptr(), 2 * B, _stream())
                if dynamic is not None:
                    rc = lib.xunet_sampler_step_dynamic(*head, hp, B, dynamic, scale.data_ptr(), *tail)
                elif hist is None:
                    rc = lib.xunet_sampler_step_table(*head, *tail)
                else:
                    rc = lib.xunet_sampler_step_multistep(*head, hp, *tail)
            else:
                rc = lib.xunet_sampler_step_cond(out.data_ptr(), z.data_ptr(), None, n, tab.data_ptr(), pos.data_ptr(),
                                                 seed.data_ptr(), hp, B, dynamic or 0.0,
                                                 scale.data_ptr() if dynamic else None, nz.data_ptr(), nl.data_ptr(),
                                                 _stream())
            assert rc == 0, lib.xunet_last_error()
            pos.add_(1)
            torch.cuda.synchronize()
            outs.append((z.clone(), nz[:n].clone(), nl[:B].clone(), scale.clone(), None if hist is None else hist.clone()))
            if guided:
                assert torch.equal(nz[:n], nz[n:]) and torch.equal(nl[:B], nl[B:])
        res[guided] = outs
    for k, (a, b) in enumerate(zip(res[True], res[False])):
        for x, y in zip(a, b):
            if x is not None:
                assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (k,)
    # bad arguments
    out = torch.zeros(n, device='cuda')
    base = lambda **kw: lib.xunet_sampler_step_cond(out.data_ptr(), z0.data_ptr(), None, kw.get('n', n), tab.data_ptr(),
                                                    pos.data_ptr(), seed.data_ptr(), None, kw.get('b', B), kw.get('p', 0.0),
                                                    None, nz.data_ptr(), nl.data_ptr(), _stream())
    for kw in (dict(n=0), dict(b=0), dict(n=n - 1), dict(p=1.5), dict(p=-0.5)):
        assert base(**kw) != 0, kw
    torch.cuda.synchronize()


def test_unguided_sampler_graph_replay_equals_eager():
    S_, B = 16, 2
    model, _, _, tree_, batch, _ = _setup(TINY, S_, B, 'bf16')
    nb = np_batch(batch)
    views, poses, K, tp = _pool_from_batch(nb)
    tp = {key: np.concatenate([tp[key], poses[key]], 1) for key in ('R', 't')}
    grid = distill_grid(16, 1)
    for method, dyn in (('ddim', None), ('ddim', 0.995), ('dpmpp_2m', None)):
        out = {}
        for use_graph in (True, False):
            samp = P.Sampler(model, tree_, B, S_, w=None, timesteps=grid, method=method, use_graph=use_graph,
                             dynamic_threshold=dyn, prediction='v')
            assert samp.eng.B == B and len(samp.sched) == len(grid)
            out[use_graph] = (samp.sample(nb, seed=3), samp.sample_views(views, poses, K, tp, seed=3))
            assert bool((samp.eng.inp['cond_mask'] == 1).all())
        assert torch.equal(out[True][0], out[False][0]) and torch.equal(out[True][1], out[False][1]), method
        assert bool(torch.isfinite(out[True][0]).all()) and bool(torch.isfinite(out[True][1]).all())
    # a guided sampler at w = 0 runs the 2B batch and is another engine
    assert P.Sampler(model, tree_, B, S_, w=0.0, timesteps=grid, method='ddim', prediction='v').eng.B == 2 * B


# ---- 7. a short distillation run learns -------------------------------------------------------------------------------------------
def test_short_distillation_run_lowers_the_loss(tree):
    S, B = 16, 4
    store = D.DeviceScenes(tree, S)
    model = P.XUNet(**dict(CFG, dropout=0.0))
    params = P.create_train_state(3, 1, 1e-3, B, S, model=model, zero_init=False).params
    teacher = Teacher(model, params, 16, batch_size=B, img_sidelength=S, w=1.0)
    st = create_distill_state(teacher, 1e-3)
    step = P.TrainStep(st, data=store, data_seed=1, teacher=teacher)
    losses = [float(step()) for _ in range(120)]
    assert np.isfinite(losses).all()
    first, last = np.mean(losses[:20]), np.mean(losses[-20:])
    assert last < 0.9 * first, (first, last)
