"""CPU checks of pose estimation: the float64 restatement of its device arithmetic (tests/pose_ref.py) against autograd, finite
differences, scipy and torch's Adam; the sphere start, rotation_error_deg and argument checks of novel_view_synthesis_3d_b200.pose;
and the helpers of examples/pose_srn.py on a synthetic scene directory."""
import importlib.util
import math
import os
import re

import cv2
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from novel_view_synthesis_3d_b200 import pose as PO
from novel_view_synthesis_3d_b200.diffusion import diffusion_tables
from novel_view_synthesis_3d_b200.srn_data import SRNScenes
from tests import pose_ref as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _random_pose(rng, r=1.3):
    R = Rotation.random(random_state=rng).as_matrix()
    t = rng.randn(3)
    return R, r * t / np.linalg.norm(t)


def _hat_t(w):
    z = torch.zeros((), dtype=w.dtype)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def _f(R, t, A, c, b):
    """a smooth function of (R, t) that couples them, as the network's loss does through the rays"""
    return torch.sin(A * R).sum() + torch.cos(c * (R @ t)).sum() + (b @ t) ** 2 + (R[0] @ t) * t[2]


@pytest.mark.parametrize('translate', [False, True])
def test_tangent_matches_autograd_and_finite_differences(translate):
    rng = np.random.RandomState(1)
    H, P = 3, 2
    A, c, b = (torch.as_tensor(x) for x in (rng.randn(3, 3), rng.randn(3), rng.randn(3)))
    poses = [_random_pose(rng) for _ in range(H)]
    dR, dt, want = [], [], []
    for R, t in poses:
        Rt, tt = torch.tensor(R, requires_grad=True), torch.tensor(t, requires_grad=True)
        G, g = torch.autograd.grad(_f(Rt, tt, A, c, b), (Rt, tt))
        # the rows' gradients of one hypothesis sum to (G, g): split them unevenly over the P draws
        parts = rng.uniform(-1, 2, P)
        parts /= parts.sum()
        dR += [G.numpy() * s for s in parts]
        dt += [g.numpy() * s for s in parts]
        D = 6 if translate else 3
        x = torch.zeros(D, dtype=torch.float64, requires_grad=True)
        E = torch.linalg.matrix_exp(_hat_t(x[:3]))
        tn = E @ torch.tensor(t) + (x[3:] if translate else 0)
        (gx,) = torch.autograd.grad(_f(E @ torch.tensor(R), tn, A, c, b), x)
        want.append(gx.numpy())
        # central differences through the reference retraction
        h, fd = 1e-6, np.zeros(D)
        for k in range(D):
            e = np.zeros(6 if translate else 3)
            e[k] = h
            Rp, tp = PR.retract(e[None], R[None], t[None], translate)
            Rm, tm = PR.retract(-e[None], R[None], t[None], translate)
            fd[k] = float(_f(torch.tensor(Rp[0]), torch.tensor(tp[0]), A, c, b) - _f(torch.tensor(Rm[0]), torch.tensor(tm[0]), A, c, b)) / (2 * h)
        assert np.allclose(fd, gx.numpy(), rtol=0, atol=1e-7 * max(1.0, np.abs(fd).max()))
    got = PR.tangent(np.stack(dR), np.stack(dt), np.stack([p[0] for p in poses]), np.stack([p[1] for p in poses]), P, translate)
    assert got.shape == (H, 6 if translate else 3)
    assert np.allclose(got, np.stack(want), rtol=1e-12, atol=1e-12)


def test_retraction_matches_scipy():
    rng = np.random.RandomState(2)
    for translate in (False, True):
        w = rng.randn(5, 6) * np.array([[0.1], [1.0], [3.0], [1e-4], [1e-9]])
        R = Rotation.random(5, random_state=rng).as_matrix()
        t = rng.randn(5, 3)
        Rn, tn = PR.retract(w if translate else w[:, :3], R, t, translate)
        E = Rotation.from_rotvec(w[:, :3]).as_matrix()
        assert np.allclose(Rn, E @ R, rtol=0, atol=1e-14)
        assert np.allclose(tn, np.einsum('hij,hj->hi', E, t) + (w[:, 3:] if translate else 0), rtol=0, atol=1e-14)
    # a zero step is the identity, exactly
    Rn, tn = PR.retract(np.zeros((5, 3)), R, t, False)
    assert np.array_equal(Rn, R) and np.array_equal(tn, t)


def test_small_angle_branch_is_continuous():
    rng = np.random.RandomState(3)
    for _ in range(20):
        u = rng.randn(3)
        u /= np.linalg.norm(u)
        th = math.sqrt(PR.SMALL_ANGLE2)
        wb, wa = u * th * (1 - 1e-12), u * th * (1 + 1e-12)        # either side of the branch point
        jump = (PR.expm_so3(wa) - PR.expm_so3(wb)) - (Rotation.from_rotvec(wa).as_matrix() - Rotation.from_rotvec(wb).as_matrix())
        assert np.abs(jump).max() < 5e-16
        for s in (0.5, 1 - 1e-9, 1 + 1e-9, 2.0):
            assert np.abs(PR.expm_so3(u * th * s) - Rotation.from_rotvec(u * th * s).as_matrix()).max() < 2e-16


def test_rotation_stays_orthonormal_over_many_steps():
    rng = np.random.RandomState(4)
    R, t = Rotation.random(random_state=rng).as_matrix()[None], np.array([[0.0, 0.0, 1.3]])
    for _ in range(10_000):
        R, t = PR.retract(rng.randn(1, 3) * 0.3, R, t, False)
    assert np.abs(R[0].T @ R[0] - np.eye(3)).max() < 1e-9
    assert abs(np.linalg.norm(t) - 1.3) < 1e-9


def test_adam_restatement_is_xunet_adam_step():
    """pose_ref.adam on a zero buffer against torch's Adam (the same update rule) in fp64, and against the fp32 arithmetic
    xunet_adam_step states (bias corrections formed in double, then rounded)"""
    rng = np.random.RandomState(5)
    lr, b1, b2, eps = 0.01, 0.9, 0.999, 1e-8
    grads = rng.randn(6, 4, 3)
    p = torch.zeros(4, 3, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([p], lr=lr, betas=(b1, b2), eps=eps)
    m = v = np.zeros((4, 3))
    m32 = v32 = np.zeros((4, 3), np.float32)
    for i, g in enumerate(grads, 1):
        before = p.detach().clone()
        p.grad = torch.as_tensor(g)
        opt.step()
        step, m, v = PR.adam(g, m, v, i, lr, b1, b2, eps)
        assert np.allclose(step, (p.detach() - before).numpy(), rtol=1e-12, atol=1e-18)
        f = np.float32
        c1, c2 = f(1.0 / (1.0 - b1 ** i)), f(1.0 / (1.0 - b2 ** i))
        g32 = g.astype(f)
        m32 = f(b1) * m32 + f(1 - b1) * g32
        v32 = f(b2) * v32 + f(1 - b2) * g32 * g32
        step32 = f(0) - f(lr) * (m32 * c1) / (np.sqrt(v32 * c2) + f(eps))
        assert np.allclose(step32, step, rtol=1e-5, atol=0)


def test_draws():
    sa, sb = diffusion_tables()
    y = np.random.RandomState(6).uniform(-1, 1, (8, 8, 3))
    H, P = 3, 4
    seen = set()
    for i in (1, 2, 3):
        t, eps, z, ls, target = PR.draw(y, H, P, seed=9, i=i, t_min=100, t_max=900, sqrt_ac=sa, sqrt_1mac=sb)
        assert np.all((t >= 100) & (t <= 900)) and t.dtype == np.int64
        # every hypothesis shares draw p
        zr = z.reshape(H, P, 8, 8, 3)
        assert all(np.array_equal(zr[0], zr[h]) for h in range(H))
        assert np.array_equal(ls.reshape(H, P)[0], ls.reshape(H, P)[2])
        assert np.array_equal(target, eps)
        assert np.allclose(zr[0], sa[t].reshape(P, 1, 1, 1) * y + sb[t].reshape(P, 1, 1, 1) * eps, atol=1e-12)
        assert abs(eps.mean()) < 0.15 and abs(eps.std() - 1) < 0.1
        seen.add(eps.tobytes())
        assert len({e.tobytes() for e in eps}) == P
    assert len(seen) == 3                    # different iterations draw differently
    assert PR.timesteps(9, 1, P, 5, 5).tolist() == [5] * P
    # v target
    t, eps, _, _, v = PR.draw(y, 1, 2, seed=9, i=1, t_min=0, t_max=999, sqrt_ac=sa, sqrt_1mac=sb, prediction='v')
    assert np.allclose(v, sa[t].reshape(2, 1, 1, 1) * eps - sb[t].reshape(2, 1, 1, 1) * y, atol=1e-12)
    # stratified: E draws over iterations 1..E/P hit each stratum once
    E = 8
    ts = np.concatenate([PR.timesteps(0, i, 2, 100, 899, strata=E) for i in range(1, E // 2 + 1)])
    assert ts.tolist() == [100 + (2 * g + 1) * 800 // (2 * E) for g in range(E)]
    assert np.all(np.diff(ts) > 0)


def test_draw_hash_restates_mix64():
    m = (1 << 64) - 1

    def mix(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
        return z ^ (z >> 31)
    assert PR.draw_hash(7, 3, 2) == mix((7 * 0x9E3779B97F4A7C15 + 3 * 0xD1B54A32D192ED03 + 2) & m)


def test_loss_and_seed():
    rng = np.random.RandomState(7)
    H, P, S = 2, 3, 4
    out, target = rng.randn(H * P, S, S, 3), rng.randn(P, S, S, 3)
    L, d = PR.loss(out, target, H, P)
    for h in range(H):
        want = np.mean([np.mean((out[h * P + p] - target[p]) ** 2) for p in range(P)])
        assert abs(L[h] - want) < 1e-14
    o = torch.tensor(out, requires_grad=True)
    Lt = ((o.reshape(H, P, -1) - torch.tensor(target).reshape(1, P, -1)) ** 2).mean(2).mean(1).sum()
    (g,) = torch.autograd.grad(Lt, o)
    assert np.allclose(d, g.reshape(H * P, -1).numpy(), rtol=1e-14, atol=0)


def test_sphere_start():
    rng = np.random.RandomState(8)
    for H in (1, 2, 7, 16):
        c = rng.randn(3)
        c = 1.7 * c / np.linalg.norm(c)
        R1 = PO.np.asarray(_look_at(c))
        R, t = PO.sphere_init(R1, c, H)
        assert R.shape == (H, 3, 3) and t.shape == (H, 3)
        assert np.allclose(R @ np.swapaxes(R, 1, 2), np.eye(3), atol=1e-12)
        assert np.allclose(np.linalg.det(R), 1.0, atol=1e-12)
        assert np.allclose(np.linalg.norm(t, axis=1), 1.7, atol=1e-12)
        # camera 1 looks at the origin (its +z axis points at -c), so every hypothesis does too
        assert np.allclose(R1[:, 2], -c / 1.7, atol=1e-12)
        assert np.allclose(R[:, :, 2], -t / 1.7, atol=1e-12)
        assert np.allclose(t / 1.7, PO.fibonacci_sphere(H), atol=1e-12)
        if H > 1:
            dots = (t @ t.T) / 1.7 ** 2
            assert dots[~np.eye(H, dtype=bool)].max() < 1 - 1e-3          # distinct directions
    # the antipodal case: t1 opposite to a lattice point
    u = PO.fibonacci_sphere(5)
    R1 = _look_at(-1.3 * u[2])
    R, t = PO.sphere_init(R1, -1.3 * u[2], 5)
    assert np.all(np.isfinite(R)) and np.allclose(t[2], 1.3 * u[2], atol=1e-12)
    assert np.allclose(R[2] @ R[2].T, np.eye(3), atol=1e-12) and abs(np.linalg.det(R[2]) - 1) < 1e-12
    assert np.allclose(R[2][:, 2], -u[2], atol=1e-12)
    for a in (np.array([1.0, 0, 0]), np.array([0, 0, -1.0]), u[0]):
        Q = PO.rotation_between(a, -a)
        assert np.allclose(Q @ a, -a, atol=1e-12) and abs(np.linalg.det(Q) - 1) < 1e-12
    with pytest.raises(ValueError, match='t1 = 0'):
        PO.sphere_init(np.eye(3), np.zeros(3), 4)


def _look_at(c):
    """cam-to-world rotation of a camera at c whose +z axis points at the origin (OpenCV: x right, y down)"""
    f = -np.asarray(c, np.float64) / np.linalg.norm(c)
    up = np.array([0.0, 0.0, 1.0]) if abs(f[2]) < 0.9 else np.array([0.0, 1.0, 0.0])
    x = np.cross(f, up)
    x /= np.linalg.norm(x)
    y = np.cross(f, x)
    return np.stack([x, y, f], 1)


def test_rotation_error_deg():
    rng = np.random.RandomState(9)
    Rb = Rotation.random(6, random_state=rng).as_matrix()
    ang = np.array([0.0, 1e-7, 5.0, 90.0, 179.0, 180.0])
    axes = rng.randn(6, 3)
    axes /= np.linalg.norm(axes, axis=1, keepdims=True)
    Ra = Rotation.from_rotvec(axes * np.radians(ang)[:, None]).as_matrix() @ Rb
    got = PO.rotation_error_deg(Ra, Rb)
    assert np.allclose(got, ang, rtol=1e-9, atol=1e-9)
    assert np.allclose(PO.rotation_error_deg(torch.as_tensor(Ra), torch.as_tensor(Rb)), ang, rtol=1e-9, atol=1e-9)
    assert float(PO.rotation_error_deg(Ra[2], Rb[2])) == pytest.approx(5.0)


@pytest.mark.parametrize('kw,msg', [
    (dict(hypotheses=0), 'hypotheses'), (dict(draws=0), 'draws'), (dict(t_range=(-1, 10)), 't_range'),
    (dict(t_range=(500, 100)), 't_range'), (dict(t_range=(0, 1000)), 't_range'), (dict(lr=-1e-3), 'lr'),
    (dict(lr=float('nan')), 'lr'), (dict(lr=float('inf')), 'lr'), (dict(prediction='x0'), 'prediction'),
    (dict(draws=2, eval_draws=3), 'eval_draws'), (dict(eval_draws=0), 'eval_draws'),
])
def test_argument_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        PO.PoseEstimator(None, None, 16, **kw)


def _defines():
    hdr = open(os.path.join(ROOT, 'include', 'xunet_b200.h')).read()
    return dict(re.findall(r'#define (XUNET_POSE_\w+) (\S+)', hdr))


def test_header_constants():
    d = _defines()
    assert int(d['XUNET_POSE_MAX_T']) == PO.MAX_T == 999
    assert int(d['XUNET_POSE_LOSS_CHUNK']) == PO.LOSS_CHUNK
    assert float(d['XUNET_POSE_SMALL_ANGLE2']) == PO.SMALL_ANGLE2 == PR.SMALL_ANGLE2


def _example():
    spec = importlib.util.spec_from_file_location('pose_srn', os.path.join(ROOT, 'examples', 'pose_srn.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_example_helpers_on_a_synthetic_scene(tmp_path):
    ex = _example()
    a = ex.parse_args([str(tmp_path), '--ckpt', 'c', '--side', '16', '--stride', '3', '--distilled', '2',
                       '--ray-convention', 'opencv_uv', '--t-range', '50', '950', '--translate'])
    assert a.side == 16 and a.stride == 3 and a.distilled == 2 and a.ray_convention == 'opencv_uv'
    assert a.t_range == [50, 950] and a.translate and a.hypotheses == PO.HYPOTHESES
    with pytest.raises(SystemExit):
        ex.parse_args([str(tmp_path), '--stride', '0'])
    # a scene directory in SRN's layout: two instances of 7 views on a sphere of radius 1.3
    rng = np.random.RandomState(10)
    for i in range(2):
        d = tmp_path / f'obj{i}'
        (d / 'rgb').mkdir(parents=True)
        (d / 'pose').mkdir()
        (d / 'intrinsics.txt').write_text('131.25 64.0 64.0 0.\n0. 0. 0.\n1.\n128 128\n')
        for v in range(7):
            cv2.imwrite(str(d / 'rgb' / f'{v:06d}.png'), rng.randint(0, 256, (32, 32, 3), dtype=np.uint8))
            c = rng.randn(3)
            c = 1.3 * c / np.linalg.norm(c)
            pose = np.eye(4)
            pose[:3, :3], pose[:3, 3] = _look_at(c), c
            (d / 'pose' / f'{v:06d}.txt').write_text(' '.join(f'{x:.9f}' for x in pose.reshape(-1)) + '\n')
    ds = SRNScenes(str(tmp_path), img_sidelength=16)
    d = ds.instance_views(1)
    targets = ex.select_targets(len(d['x']), 4, 3)
    assert targets == [0, 3, 6]
    assert ex.select_targets(7, 3, 3) == [0, 6]
    e = ex.pair_errors(d['R'][0], d['t'][0], d['R'][0], d['t'][0])
    assert e['rot_err_deg'] < 1e-5 and e['center_err'] == 0.0
    recs = [ex.pair_errors(d['R'][v], d['t'][v], d['R'][0], d['t'][0]) for v in range(7)]
    want = PO.rotation_error_deg(d['R'], d['R'][0])
    assert np.allclose([r['rot_err_deg'] for r in recs], want)
    s = ex.summarize(recs)
    assert s['n_pairs'] == 7 and s['median_rot_err_deg'] == pytest.approx(float(np.median(want)))
    assert s['acc_15'] == pytest.approx(float(np.mean(want < 15))) and s['acc_30'] == pytest.approx(float(np.mean(want < 30)))
    assert ex.summarize([])['n_pairs'] == 0
