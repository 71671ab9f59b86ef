"""Consistency distillation on the GPU: xunet_cd_teacher_step against xunet_sampler_step_table / _cond at pos = m, the target
kernel against an fp32 numpy restatement, a train=0 forward on the training engine leaving the next train step's bits
alone, the captured consistency-distillation TrainStep against an eager composition, the consistency sampler against a
numpy restatement of its table steps, and a short run with its checkpoint record."""
import ctypes as C

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip('cv2')
import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200 import checkpoint as ck
from novel_view_synthesis_3d_b200 import srn_data as D
from novel_view_synthesis_3d_b200.distill import ConsistencyTeacher, cd_target_table, create_distill_state
from novel_view_synthesis_3d_b200.sampling import Schedule, consistency_grid, distill_grid, sampler_table
from novel_view_synthesis_3d_b200.xunet import InputSlots
from tests.test_gpu_device_data import CFG, _write_tree
from tests.test_gpu_distill import BATCH_KEYS, _fma, _teacher_model_params
from tests.test_gpu_model import _pool_from_batch, _setup
from tests.test_gpu_v_prediction import TINY, _bits, _nan, _stream, _tables
from tests.util import np_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return _write_tree(tmp_path_factory.mktemp('srn_cd'))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---- 1. the teacher step is the sampler step at pos = m -------------------------------------------------------------------------
@pytest.mark.parametrize('copies,pred', [(2, 'eps'), (1, 'eps'), (1, 'v'), (2, 'v')])
def test_cd_teacher_step_is_the_sampler_step_at_m(lib, copies, pred):
    B, S, w, N = 6, 8, 2.5, 32
    per = S * S * 3
    n = B * per
    tab = _dev(sampler_table(Schedule(timesteps=distill_grid(N, 0)), 'ddim', prediction=pred,
                             logsnr_lag=False)[0].astype(np.float32))
    g = torch.Generator(device='cuda').manual_seed(3)
    out = torch.randn(copies * n, generator=g, device='cuda') * 1.5
    z_t = torch.randn(n, generator=g, device='cuda')
    z_keep = z_t.clone()
    m = torch.tensor([0, N - 1, 7, 3, N - 1, 30], dtype=torch.int32, device='cuda')     # mixed, with the last row
    z_buf, l_buf = _nan(n + 64), _nan(B + 8)              # the tails must stay untouched
    assert lib.xunet_cd_teacher_step(out.data_ptr(), w, copies, tab.data_ptr(), m.data_ptr(), B, per, z_t.data_ptr(),
                                     z_buf.data_ptr(), l_buf.data_ptr(), _stream()) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    assert torch.equal(z_t.view(torch.int32), z_keep.view(torch.int32))
    assert bool(torch.isnan(z_buf[n:]).all()) and bool(torch.isnan(l_buf[B:]).all())
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    for b in range(B):
        sl = slice(b * per, (b + 1) * per)
        z = z_keep[sl].clone()
        pos = torch.full((1,), int(m[b]), dtype=torch.int32, device='cuda')
        if copies == 2:
            o2 = torch.cat([out[sl], out[n + b * per:n + (b + 1) * per]])
            nz, nl = torch.zeros(2 * per, device='cuda'), torch.zeros(2, device='cuda')
            assert lib.xunet_sampler_step_table(o2.data_ptr(), z.data_ptr(), None, per, w, tab.data_ptr(), pos.data_ptr(),
                                                seed.data_ptr(), nz.data_ptr(), nl.data_ptr(), 2, _stream()) == 0
        else:
            o1 = out[sl].clone()
            nz, nl = torch.zeros(per, device='cuda'), torch.zeros(1, device='cuda')
            assert lib.xunet_sampler_step_cond(o1.data_ptr(), z.data_ptr(), None, per, tab.data_ptr(), pos.data_ptr(),
                                               seed.data_ptr(), None, 1, 0.0, None, nz.data_ptr(), nl.data_ptr(),
                                               _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(z_buf[sl].view(torch.int32), z.view(torch.int32)), b
        assert l_buf[b].item() == tab[int(m[b]), 5].item() == nl[0].item()
    # argument errors
    def call(out=out.data_ptr(), copies=copies, tab=tab.data_ptr(), m=m.data_ptr(), B=B, per=per, z=z_t.data_ptr(),
             zo=z_buf.data_ptr(), lo=l_buf.data_ptr()):
        return lib.xunet_cd_teacher_step(out, w, copies, tab, m, B, per, z, zo, lo, _stream())
    for kw in (dict(out=None), dict(tab=None), dict(m=None), dict(z=None), dict(zo=None), dict(lo=None), dict(B=0),
               dict(per=0), dict(copies=3), dict(copies=0)):
        assert call(**kw) != 0, kw
        assert 'xunet_cd_teacher_step' in lib.xunet_last_error().decode()
    torch.cuda.synchronize()


# ---- 2. the target kernel against an fp32 numpy restatement -----------------------------------------------------------------------
def test_cd_target_matches_numpy(lib):
    B, S, N = 5, 8, 40
    per = S * S * 3
    n = B * per
    gtab = cd_target_table(distill_grid(N, 0)).astype(np.float32)
    r = np.random.RandomState(4)
    vm = (r.randn(n) * 0.7).astype(np.float32)
    zh = (r.randn(n) * 0.8).astype(np.float32)
    zt = r.randn(n).astype(np.float32)
    m = np.array([0, N - 1, 4, 20, N - 1], np.int32)
    v = _nan(n)
    assert lib.xunet_cd_target(_dev(vm).data_ptr(), _dev(gtab).data_ptr(), _dev(m).data_ptr(), _dev(zt).data_ptr(),
                               _dev(zh).data_ptr(), B, per, v.data_ptr(), _stream()) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    g = gtab[np.repeat(m, per)]
    f = np.float32
    x0 = np.clip(_fma(g[:, 0], zh, -(g[:, 1] * vm)), f(-1), f(1))
    want = ((g[:, 2] * zt) - x0) / g[:, 3]
    assert np.array_equal(_bits(v), want.astype(np.float32).view(np.int32))
    last = np.repeat(m == N - 1, per)
    np.testing.assert_array_equal(x0[last], np.clip(zh[last], -1, 1))    # the boundary: x0- = z^
    args = [_dev(vm).data_ptr(), _dev(gtab).data_ptr(), _dev(m).data_ptr(), _dev(zt).data_ptr(), _dev(zh).data_ptr()]
    for i in range(5):
        bad = list(args)
        bad[i] = None
        assert lib.xunet_cd_target(*bad, B, per, v.data_ptr(), _stream()) != 0
    assert lib.xunet_cd_target(*args, B, per, None, _stream()) != 0
    assert lib.xunet_cd_target(*args, 0, per, v.data_ptr(), _stream()) != 0
    assert lib.xunet_cd_target(*args, B, 0, v.data_ptr(), _stream()) != 0
    assert 'xunet_cd_target' in lib.xunet_last_error().decode()
    torch.cuda.synchronize()


# ---- 3. a train=0 forward on the training engine leaves the next train step alone -------------------------------------------------
@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
def test_train0_forward_before_a_train_step_changes_no_bit(dtype):
    """The target forward of a consistency-distillation step runs on the student's training engine, with other z and
    log-SNR inputs, right before the student's train forward (dropout on): that forward's output, the mse loss and the
    parameter gradient are those of the same step without it."""
    S, B = 16, 4
    model = P.XUNet(**CFG, dtype=dtype)
    st = P.create_train_state(0, 1, 1e-3, B, S, model=model, zero_init=False, loss='mse', prediction='v')
    eng = model.engine(B, S, True)
    data = P.create_sample_data(B, S)
    noise = data.pop('noise')
    eng.load_inputs(data, cond_mask=np.ones(B, np.float32), noise=noise)
    g = torch.Generator(device='cuda').manual_seed(9)
    z2, l2 = torch.randn(B, S, S, 3, generator=g, device='cuda'), torch.rand(B, generator=g, device='cuda') * 10 - 5
    cb = _lib.XunetBatch.from_buffer_copy(eng.cbatch)
    cb.z, cb.logsnr = z2.data_ptr(), l2.data_ptr()
    res = []
    for before in (False, True, False):
        vm = _nan(B * S * S * 3).view(B, S, S, 3)
        if before:
            y = eng.forward(st.params.flat, train=False, batch=cb, out=vm)
            assert y is vm
        eps = eng.forward(st.params.flat, train=True, seed=77).clone()
        loss, grads = eng.backward(st.params.flat, loss='mse')
        torch.cuda.synchronize()
        res.append((eps, loss.clone(), grads.clone(), vm.clone()))
        if before:
            assert bool(torch.isfinite(vm).all()) and not torch.equal(vm, eps)
    for a in res[1:]:
        for x, y in zip(res[0][:3], a[:3]):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    with pytest.raises(ValueError, match='out must'):
        eng.forward(st.params.flat, train=False, out=torch.zeros(B, S, S, 3, device='cuda', dtype=torch.float64))


# ---- 4. the captured consistency-distillation step equals the eager composition -----------------------------------------------
@pytest.mark.parametrize('k,w', [(1, 3.0), (2, None), (1, None), (2, 3.0)])
def test_captured_cd_step_equals_the_eager_composition(tree, lib, k, w):
    S, B, seed, N = 16, 4, 21, 24
    store = D.DeviceScenes(tree, S)
    model, params = _teacher_model_params(S, B)
    # two model objects: the two students must not share an engine (and so a gradient buffer)
    ta = ConsistencyTeacher(model, params, N, batch_size=B, img_sidelength=S, w=w)
    tb = ConsistencyTeacher(P.XUNet(**CFG), params, N, batch_size=B, img_sidelength=S, w=w)
    sa, sb = create_distill_state(ta, 1e-3), create_distill_state(tb, 1e-3)
    assert sa.distill == ta.record == ({'cd_steps': N} if w is None else {'cd_steps': N, 'w': w})
    assert torch.equal(sa.params.flat, ta.flat) and sa.prediction == 'v' and sa.loss == 'mse'
    step_a = P.TrainStep(sa, data=store, data_seed=seed, grad_accum_steps=k, teacher=ta)
    step_b = P.TrainStep(sb, grad_accum_steps=k)
    assert step_b.eng is not step_a.eng
    slots = InputSlots(B, S, 1, store.device)
    per = S * S * 3
    st = _stream()
    z_hat, l_hat, v_minus = _nan(B * per), _nan(B), _nan(B * per)
    for c in range(3):
        parts = []
        for j in range(k):
            step_dev = torch.full((1,), c + 1, dtype=torch.int64, device='cuda')
            sqa, sqb = _tables()
            assert lib.xunet_srn_batch_distill(C.byref(store.c_store), step_dev.data_ptr(), seed, j, k, 0, 1, B,
                                               sqa.data_ptr(), sqb.data_ptr(), tb.grid_t.data_ptr(), N,
                                               C.byref(slots.cbatch[0]), C.byref(tb.eng.cbatch), tb.copies, tb.m.data_ptr(),
                                               None, None, st) == 0
            tb.eng.forward(tb.flat, train=False)
            zt = slots.inp[0]['z']
            assert lib.xunet_cd_teacher_step(tb.eng.eps.data_ptr(), w or 0.0, tb.copies, tb.table.data_ptr(),
                                             tb.m.data_ptr(), B, per, zt.data_ptr(), z_hat.data_ptr(), l_hat.data_ptr(),
                                             st) == 0
            cb = _lib.XunetBatch.from_buffer_copy(slots.cbatch[0])
            cb.z, cb.logsnr = z_hat.data_ptr(), l_hat.data_ptr()
            assert lib.xunet_forward(step_b.eng.h, sb.params.flat.data_ptr(), C.byref(cb), 0, None, step_b.eng.ws.data_ptr(),
                                     v_minus.data_ptr(), st) == 0
            assert lib.xunet_cd_target(v_minus.data_ptr(), tb.target.data_ptr(), tb.m.data_ptr(), zt.data_ptr(),
                                       z_hat.data_ptr(), B, per, slots.inp[0]['noise'].data_ptr(), st) == 0
            parts.append({key: slots.inp[0][key].clone() for key in BATCH_KEYS + ('cond_mask', 'noise')})
        cat = lambda key: torch.cat([p[key] for p in parts]).clone()
        batch = {key: cat(key) for key in BATCH_KEYS}
        assert bool((cat('cond_mask') == 1).all()) and bool(torch.isfinite(cat('noise')).all())
        la = float(step_a())
        lb = float(step_b(batch, cat('noise'), cond_mask=cat('cond_mask')))
        torch.cuda.synchronize()
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32), (c, la, lb)
        assert torch.equal(step_a.eng.grads.view(torch.int32), step_b.eng.grads.view(torch.int32)), c
        assert torch.equal(ta.z_hat.view(-1).view(torch.int32), z_hat.view(torch.int32)), c
        assert torch.equal(ta.v_minus.view(-1).view(torch.int32), v_minus.view(torch.int32)), c
    for x, y in ((sa.params.flat, sb.params.flat), (sa.opt_state.mu, sb.opt_state.mu), (sa.opt_state.nu, sb.opt_state.nu)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert step_a.mode == 'one_graph' and step_a.h2d_bytes == 0
    # the same step run eagerly, and replayed in a second captured step, gives the same bits
    sc = create_distill_state(tb, 1e-3)
    step_c = P.TrainStep(sc, data=store, data_seed=seed, grad_accum_steps=k, teacher=tb, use_graph=False)
    sd = create_distill_state(ta, 1e-3)
    step_d = P.TrainStep(sd, data=store, data_seed=seed, grad_accum_steps=k, teacher=ta)
    for c in range(2):
        lc, ld = float(step_c()), float(step_d())
        assert np.float32(lc).view(np.int32) == np.float32(ld).view(np.int32), c
    torch.cuda.synchronize()
    assert torch.equal(sc.params.flat.view(torch.int32), sd.params.flat.view(torch.int32))


# ---- 5. the consistency sampler ------------------------------------------------------------------------------------------------------
def test_consistency_sampler_graph_replay_and_numpy():
    S_, B, N = 16, 2, 64
    model, _, _, tree_, batch, _ = _setup(TINY, S_, B, 'bf16')
    nb = np_batch(batch)
    views, poses, K, tp = _pool_from_batch(nb)
    tp = {key: np.concatenate([tp[key], poses[key]], 1) for key in ('R', 't')}
    r = np.random.RandomState(5)
    for k in (1, 2, 4):
        ts = consistency_grid(N, k)
        z_init = r.randn(B, S_, S_, 3).astype(np.float32)
        noises = r.randn(k, B, S_, S_, 3).astype(np.float32)
        out = {}
        for use_graph in (True, False):
            samp = P.Sampler(model, tree_, B, S_, w=None, timesteps=ts, method='consistency', prediction='v',
                             use_graph=use_graph)
            assert samp.eng.B == B and len(samp.sched) == k and not samp.logsnr_lag
            outs = []
            if not use_graph:
                fwd = samp.eng.forward

                def rec(*a, **kw):
                    y = fwd(*a, **kw)
                    outs.append(y.detach().cpu().numpy().reshape(-1).copy())
                    return y
                samp.eng.forward = rec
            out[use_graph] = (samp.sample(nb, z_init=z_init, noises=noises), samp.sample(nb, seed=3),
                              samp.sample_views(views, poses, K, tp, seed=3))
            if not use_graph:
                del samp.eng.forward
        for a, b in zip(out[True], out[False]):
            assert torch.equal(a, b), k
            assert bool(torch.isfinite(a).all())
        # the table steps restated in numpy on the engine's outputs (the first sample of the eager sampler)
        rows = sampler_table(Schedule(timesteps=ts), 'consistency', prediction='v')[0].astype(np.float32)
        z = z_init.reshape(-1)
        for j in range(k):
            t = rows[j]
            x0 = np.clip(_fma(t[0], z, -(t[1] * outs[j])), np.float32(-1), np.float32(1))
            z = _fma(t[4], noises[j].reshape(-1), _fma(t[2], x0, t[3] * z))
        assert np.array_equal(_bits(out[False][0]).reshape(-1), z.view(np.int32)), k
    # dynamic thresholding runs the same rows
    dyn = [P.Sampler(model, tree_, B, S_, w=None, timesteps=consistency_grid(N, 2), method='consistency', prediction='v',
                     dynamic_threshold=0.995, use_graph=g).sample(nb, seed=1) for g in (True, False)]
    assert torch.equal(dyn[0], dyn[1]) and bool(torch.isfinite(dyn[0]).all())


# ---- 6. a short consistency-distillation run learns, and its record round-trips ---------------------------------------------------
def test_short_cd_run_lowers_the_loss_and_checkpoints(tree, tmp_path):
    S, B = 16, 4
    store = D.DeviceScenes(tree, S)
    model = P.XUNet(**dict(CFG, dropout=0.0))
    params = P.create_train_state(3, 1, 1e-3, B, S, model=model, zero_init=False).params
    teacher = ConsistencyTeacher(model, params, 16, batch_size=B, img_sidelength=S, w=1.0)
    st = create_distill_state(teacher, 1e-3)
    step = P.TrainStep(st, data=store, data_seed=1, teacher=teacher)
    losses = [float(step()) for _ in range(120)]
    assert np.isfinite(losses).all()
    first, last = np.mean(losses[:20]), np.mean(losses[-20:])
    assert last < 0.9 * first, (first, last)
    ck.save_train_state(str(tmp_path), st, step=st.step)
    dst = create_distill_state(teacher, 1e-3)
    assert dst.distill == {'cd_steps': 16, 'w': 1.0}
    assert ck.restore_train_state(str(tmp_path), dst) is dst
    assert torch.equal(dst.params.flat, st.params.flat) and dst.step == st.step
    other = create_distill_state(ConsistencyTeacher(model, params, 16, batch_size=B, img_sidelength=S, w=None), 1e-3)
    with pytest.raises(ValueError, match='distillation record'):
        ck.restore_train_state(str(tmp_path), other)
