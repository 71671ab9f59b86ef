"""Pose estimation on the GPU (csrc/pose_fit.cu, pose.PoseEstimator): each kernel against the float64 restatement of
tests/pose_ref.py, one replayed iteration against the same iteration composed eagerly from the public engine calls, the
tangent gradient against finite differences of the evaluation loss, fixed bits, a bf16 run of the small model, and errors."""

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as NV
from novel_view_synthesis_3d_b200 import pose as PO
from novel_view_synthesis_3d_b200.diffusion import diffusion_tables
from tests import pose_ref as PR
from tests.test_pose_cpu import _look_at

pytestmark = pytest.mark.gpu

SMALL = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=2, attn_resolutions=(8, 16, 32), attn_heads=4, dropout=0.0)
TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _views(S, seed=0):
    """x, R1, t1, K, y: two smooth random views and a camera 1 on the sphere of radius 1.3 looking at the origin"""
    g = torch.Generator().manual_seed(seed)
    lo = torch.rand(2, 3, 4, 4, generator=g) * 2 - 1
    v = torch.nn.functional.interpolate(lo, size=(S, S), mode='bilinear', align_corners=False).permute(0, 2, 3, 1)
    c = np.array([0.3, -0.8, 0.9])
    c = 1.3 * c / np.linalg.norm(c)
    f = 131.25 * S / 128
    K = np.array([[f, 0, S / 2], [0, f, S / 2], [0, 0, 1.0]])
    return v[0].numpy(), _look_at(c), c, K, v[1].numpy()


def _estimator(cfg, dtype, S, H, P, **kw):
    model = NV.XUNet(**cfg, dtype=dtype)
    params = model.init({'params': 0}, {'x': np.zeros((1, S, S, 3))}, zero_init=False)['params']
    return PO.PoseEstimator(model, params, S, hypotheses=H, draws=P, **kw)


def _cpu(t):
    return t.detach().cpu().double().numpy()


# ---- 1. the draw -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prediction,strata', [('eps', 0), ('v', 0), ('eps', 6)])
def test_draw_kernel_matches_reference(lib, prediction, strata):
    H, P, S, seed = 3, 2, 20, 77
    sa, sb = diffusion_tables()
    sa_d, sb_d = torch.as_tensor(sa).cuda(), torch.as_tensor(sb).cuda()
    y = torch.rand(S, S, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1
    yd = y.cuda()
    z = torch.zeros(H * P, S, S, 3, device='cuda')
    ls = torch.zeros(H * P, device='cuda')
    tg = torch.zeros(P, S, S, 3, device='cuda')
    tt = torch.zeros(P, dtype=torch.int32, device='cuda')
    for i in (1, 2, 3):
        it = torch.tensor([i], dtype=torch.int64, device='cuda')
        assert lib.xunet_pose_draw(yd.data_ptr(), H, P, S, 40, 960, strata, it.data_ptr(), seed, sa_d.data_ptr(), sb_d.data_ptr(),
                                   int(prediction == 'v'), z.data_ptr(), ls.data_ptr(), tg.data_ptr(), tt.data_ptr(),
                                   _stream()) == 0, lib.xunet_last_error()
        t, eps, zr, lr, target = PR.draw(y.numpy(), H, P, seed, i, 40, 960, sa, sb, prediction, strata)
        torch.cuda.synchronize()
        assert tt.cpu().tolist() == t.tolist()
        # fp32 Box-Muller: the argument 2 pi u2 is rounded once, a few 1e-7 of the angle times |normal| <= 5.8
        assert np.allclose(_cpu(tg), target, rtol=1e-5, atol=1e-5)
        assert np.allclose(_cpu(z), zr, rtol=1e-5, atol=1e-5)
        assert np.allclose(_cpu(ls), lr, rtol=1e-6, atol=1e-6)
        zz = z.view(H, P, -1)
        assert torch.equal(zz[0], zz[H - 1])          # common random numbers, bit for bit


# ---- 2. the loss and its seed ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,P,S', [(2, 3, 20), (3, 2, 64), (1, 1, 8)])
def test_loss_kernel_matches_fp64(lib, H, P, S):
    g = torch.Generator().manual_seed(H * 100 + S)
    out = torch.randn(H * P, S, S, 3, generator=g)
    tgt = torch.randn(P, S, S, 3, generator=g)
    od, td = out.cuda(), tgt.cuda()
    d = torch.zeros_like(od)
    part = torch.zeros(H * P * -(-3 * S * S // PO.LOSS_CHUNK), dtype=torch.float64, device='cuda')
    hist = torch.full((3, H), -1.0, device='cuda')
    it = torch.tensor([2], dtype=torch.int64, device='cuda')
    runs = []
    for _ in range(2):
        assert lib.xunet_pose_loss(od.data_ptr(), td.data_ptr(), H, P, S, it.data_ptr(), part.data_ptr(), d.data_ptr(),
                                   hist.data_ptr(), 3, _stream()) == 0, lib.xunet_last_error()
        runs.append((hist.clone(), d.clone()))
    L, dref = PR.loss(out.numpy(), tgt.numpy(), H, P)
    h = _cpu(runs[0][0])
    assert np.all(h[0] == -1) and np.all(h[2] == -1)      # only row i - 1 is written
    assert np.abs(h[1] / L - 1).max() < 1e-6
    dd = _cpu(runs[0][1]).reshape(H * P, -1)
    assert np.abs(dd - dref).max() <= 1e-6 * np.abs(dref).max()
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


# ---- 3. tangent, Adam, retraction ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('translate', [False, True])
def test_tangent_adam_retract_match_fp64(lib, translate):
    H, P = 5, 3
    rng = np.random.RandomState(3)
    from scipy.spatial.transform import Rotation
    R = Rotation.random(H, random_state=rng).as_matrix()
    t = rng.randn(H, 3)
    dR, dt = rng.randn(H * P, 3, 3).astype(np.float32), rng.randn(H * P, 3).astype(np.float32)
    D = 6 if translate else 3
    Rd, td = torch.as_tensor(R).cuda(), torch.as_tensor(t).cuda()
    grad = torch.zeros(H, D, device='cuda')
    step, m, v = torch.zeros(H, D, device='cuda'), torch.zeros(H, D, device='cuda'), torch.zeros(H, D, device='cuda')
    rows_R, rows_t = torch.zeros(H * P, 3, 3, device='cuda'), torch.zeros(H * P, 3, device='cuda')
    dRd, dtd = torch.as_tensor(dR).cuda(), torch.as_tensor(dt).cuda()
    count = torch.ones(1, dtype=torch.int64, device='cuda')
    mr, vr = np.zeros((H, D)), np.zeros((H, D))
    for i in (1, 2):
        count.fill_(i)
        assert lib.xunet_pose_tangent(dRd.data_ptr(), dtd.data_ptr(), H, P, Rd.data_ptr(), td.data_ptr(), int(translate),
                                      grad.data_ptr(), _stream()) == 0, lib.xunet_last_error()
        assert lib.xunet_adam_step(step.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), H * D, 0, count.data_ptr(),
                                   0.05, 0.9, 0.999, 1e-8, 1.0, _stream()) == 0
        stp = _cpu(step)
        assert lib.xunet_pose_retract(step.data_ptr(), H, P, int(translate), Rd.data_ptr(), td.data_ptr(), rows_R.data_ptr(),
                                      rows_t.data_ptr(), _stream()) == 0, lib.xunet_last_error()
        gref = PR.tangent(dR, dt, R, t, P, translate)
        assert np.abs(_cpu(grad) - gref).max() <= 1e-6 * np.abs(gref).max()
        sref, mr, vr = PR.adam(_cpu(grad), mr, vr, i, 0.05)
        assert np.abs(stp - sref).max() <= 1e-6 * np.abs(sref).max()
        R, t = PR.retract(stp, R, t, translate)
        assert np.abs(_cpu(Rd) - R).max() < 1e-14 and np.abs(_cpu(td) - t).max() < 1e-14
        assert np.abs(_cpu(rows_R).reshape(H, P, 3, 3) - R[:, None]).max() < 1e-6
        assert np.abs(_cpu(rows_t).reshape(H, P, 3) - t[:, None]).max() < 1e-6
        assert torch.count_nonzero(step) == 0
        R, t = _cpu(Rd), _cpu(td)              # continue from the device's masters


# ---- 4. one replayed iteration against the eager composition ---------------------------------------------------------------
def test_graph_iteration_equals_eager_composition(lib):
    S, H, P = 16, 2, 2
    est = _estimator(TINY, 'bf16', S, H, P, lr=0.02)
    x, R1, t1, K, y = _views(S)
    a = est.estimate(x, R1, t1, K, y, iters=2, seed=5)
    dR2, dt2, grad2 = est.dR.clone(), est.dt.clone(), est.grad.clone()
    # the same first iteration again, then the second one by hand
    est.estimate(x, R1, t1, K, y, iters=1, seed=5)
    R, t, m, v = _cpu(est.R), _cpu(est.t), _cpu(est.m), _cpu(est.v)
    assert int(est.count.item()) == 2
    hist = torch.zeros(2, H, device='cuda')
    est._draw(est.count.data_ptr(), 5, 0)
    out = est.eng.forward(est.flat, train=False, inputs=(est.slots, 0))
    assert lib.xunet_pose_loss(out.data_ptr(), est.target.data_ptr(), H, P, S, est.count.data_ptr(), est.partial.data_ptr(),
                               est.d_eps.data_ptr(), hist.data_ptr(), 2, _stream()) == 0
    _, g = est.eng.backward_vjp_inputs(est.flat, est.d_eps, cameras=True, inputs=(est.slots, 0))
    assert torch.equal(hist[1], a.loss[1])
    assert torch.equal(g['R2'], dR2) and torch.equal(g['t2'], dt2)
    gref = PR.tangent(_cpu(g['R2']), _cpu(g['t2']), R, t, P, False)
    assert np.abs(_cpu(grad2) - gref).max() <= 1e-6 * np.abs(gref).max()
    step, _, _ = PR.adam(_cpu(grad2), m, v, 2, 0.02)
    Rr, tr = PR.retract(step, R, t, False)
    assert np.abs(_cpu(a.R) - Rr).max() < 1e-7 and np.abs(_cpu(a.t) - tr).max() < 1e-7


# ---- 5. the chain rule end to end ----------------------------------------------------------------------------------------------
# posenc channels of the scales k <= 1 (pos: 15 scales, dir: 8; [raw xyz | sin_k xyz | shifted sin_k xyz] per ray part)
LOW = [c for base, nd in ((0, 15), (93, 8)) for c in [base + d for d in range(3)] +
       [base + 3 + off + 3 * k + d for off in (0, 3 * nd) for k in range(2) for d in range(3)]]


@pytest.mark.parametrize('translate', [False, True])
def test_tangent_gradient_matches_finite_differences_of_the_score(translate):
    """The pose embedding of a fresh network reads ray positions at scales up to 2^14 (a period of 4e-4 scene units), far below
    any step a central difference of an fp32 network can take; the check zeroes the pose-embedding weights of every posenc
    channel above scale 2, which leaves the loss smooth in the pose at the scale of the step and the chain rule unchanged."""
    S, H, P = 16, 2, 2
    model = NV.XUNet(**TINY, dtype='fp32')
    params = model.init({'params': 0}, {'x': np.zeros((1, S, S, 3))}, zero_init=False)['params']
    high = torch.ones(144, dtype=torch.bool)
    high[LOW] = False
    for conv in ('Conv_0', 'Conv_1'):
        params['ConditioningProcessor_0'][conv]['kernel'][..., high, :] = 0.0
    est = PO.PoseEstimator(model, params, S, hypotheses=H, draws=P, translate=translate, eval_draws=2, t_range=(200, 600))
    x, R1, t1, K, y = _views(S, seed=1)
    est.estimate(x, R1, t1, K, y, iters=1)
    R0, t0 = PO.sphere_init(R1, t1, H)
    _, g = est.score(R0, t0, grad=True)
    g = _cpu(g)
    D = 6 if translate else 3

    def central(h):
        fd = np.zeros((H, D))
        for k in range(D):
            e = np.zeros((H, D))
            e[:, k] = h
            fd[:, k] = (_cpu(est.score(*PR.retract(e, R0, t0, translate))) -
                        _cpu(est.score(*PR.retract(-e, R0, t0, translate)))) / (2 * h)
        return fd

    fd = (4 * central(1e-2) - central(2e-2)) / 3          # Richardson: truncation O(h^4)
    for j in range(H):
        assert np.linalg.norm(g[j]) > 1e-3, g[j]                 # the check is not vacuous
        assert np.linalg.norm(fd[j] - g[j]) < 1e-3 * np.linalg.norm(g[j]), (j, fd[j], g[j])


# ---- 6. determinism --------------------------------------------------------------------------------------------------------
def test_fixed_bits_graph_and_eager():
    S, H, P = 16, 3, 2
    est = _estimator(TINY, 'bf16', S, H, P, lr=0.05, translate=True)
    x, R1, t1, K, y = _views(S, seed=2)
    runs = [est.estimate(x, R1, t1, K, y, iters=6, seed=11, use_graph=ug) for ug in (True, True, False)]
    for r in runs[1:]:
        for f in ('R', 't', 'score', 'loss'):
            assert torch.equal(getattr(runs[0], f), getattr(r, f)), f
    assert not torch.equal(runs[0].loss[0], runs[0].loss[1])           # each iteration draws afresh
    other = est.estimate(x, R1, t1, K, y, iters=6, seed=12)
    assert not torch.equal(other.loss, runs[0].loss)
    R0, t0 = PO.sphere_init(R1, t1, H)
    assert not np.allclose(_cpu(runs[0].R), R0)                        # the poses moved


def test_zero_lr_keeps_the_start():
    S, H, P = 16, 2, 2
    est = _estimator(TINY, 'bf16', S, H, P, lr=0.0, translate=True)
    x, R1, t1, K, y = _views(S, seed=3)
    R0 = torch.tensor(PO.sphere_init(R1, t1, H)[0]) @ torch.tensor(_look_at([0.0, 0.0, 1.0])).T
    t0 = torch.tensor([[0.1, 0.2, 1.2], [-0.5, 0.3, -1.1]], dtype=torch.float64)
    res = est.estimate(x, R1, t1, K, y, iters=5, init=(R0, t0))
    assert torch.equal(res.R.cpu(), R0) and torch.equal(res.t.cpu(), t0)
    assert torch.equal(res.score, est.score(R0, t0))


# ---- 7. the small model in bf16 --------------------------------------------------------------------------------------------
def test_small_bf16_smoke():
    S, H, P = 64, 4, 2
    est = _estimator(SMALL, 'bf16', S, H, P, lr=0.02)
    x, R1, t1, K, y = _views(S, seed=4)
    res = est.estimate(x, R1, t1, K, y, iters=20)
    for f in ('R', 't', 'score', 'loss'):
        assert torch.isfinite(getattr(res, f)).all(), f
    R = _cpu(res.R)
    assert np.abs(R @ np.swapaxes(R, 1, 2) - np.eye(3)).max() < 1e-5
    assert np.abs(np.linalg.det(R) - 1).max() < 1e-5
    assert 0 <= res.best < H and torch.equal(res.R_best, res.R[res.best])
    assert np.allclose(np.linalg.norm(_cpu(res.t), axis=1), np.linalg.norm(np.float32(t1)), atol=1e-12)   # rotation only: on the sphere
    err = PO.rotation_error_deg(res.R, res.R_best)
    assert err[res.best] < 1e-6


# ---- 8. errors ------------------------------------------------------------------------------------------------------------------
def test_errors(lib):
    S, H, P = 16, 2, 2
    est = _estimator(TINY, 'bf16', S, H, P)
    x, R1, t1, K, y = _views(S)
    with pytest.raises(ValueError, match='rays'):
        est.estimate(x, R1, t1, K, y, iters=2, rays=np.zeros((H * P, 2, S, S, 6), np.float32))
    with pytest.raises(ValueError, match='x'):
        est.estimate(x[:8], R1, t1, K, y)
    with pytest.raises(ValueError, match='y'):
        est.estimate(x, R1, t1, K, y[None])
    with pytest.raises(ValueError, match='K'):
        est.estimate(x, R1, t1, K[:2], y)
    with pytest.raises(ValueError, match='iters'):
        est.estimate(x, R1, t1, K, y, iters=0)
    with pytest.raises(ValueError, match='hypotheses'):      # H P other than the engine's batch
        est.estimate(x, R1, t1, K, y, init=PO.sphere_init(R1, t1, H + 1))
    with pytest.raises(ValueError, match='hypotheses'):
        est.score(*PO.sphere_init(R1, t1, 1))
    with pytest.raises(ValueError, match='init'):
        est.estimate(x, R1, t1, K, y, init='grid')
    model = NV.XUNet(**TINY)
    for tr in ((-1, 5), (10, 1000), (7, 3)):
        with pytest.raises(ValueError, match='t_range'):
            PO.PoseEstimator(model, None, S, t_range=tr)
    # the C entries check before they launch
    buf = torch.zeros(4096, device='cuda')
    it = torch.ones(1, dtype=torch.int64, device='cuda')
    p = buf.data_ptr()
    assert lib.xunet_pose_draw(p, 1, 1, 4, 0, 1000, 0, it.data_ptr(), 0, p, p, 0, p, p, p, None, _stream()) != 0
    assert b't range' in lib.xunet_last_error()
    assert lib.xunet_pose_draw(p, 0, 1, 4, 0, 10, 0, it.data_ptr(), 0, p, p, 0, p, p, p, None, _stream()) != 0
    assert lib.xunet_pose_draw(p, 1, 1, 4, 0, 10, 0, it.data_ptr(), 0, p, p, 2, p, p, p, None, _stream()) != 0
    assert lib.xunet_pose_loss(p, p, 1, 1, 4, it.data_ptr(), None, p, p, 1, _stream()) != 0
    assert lib.xunet_pose_tangent(p, p, 1, 1, p, p, 2, p, _stream()) != 0
    assert lib.xunet_pose_retract(p, 1, 0, 0, p, p, p, p, _stream()) != 0
    torch.cuda.synchronize()
