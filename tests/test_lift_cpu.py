"""CPU checks of lifting (novel_view_synthesis_3d_b200.lift and its fp64 restatement tests/lift_ref.py): the drawn cameras,
the look-at with its fallback, estimate_up / elevation_range, the v-to-eps conversion, the render backward against central
differences, the header's constants, argument errors and the helpers of examples/lift_srn.py on a synthetic scene directory."""
import importlib.util
import math
import os
import re

import cv2
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from novel_view_synthesis_3d_b200 import lift as LI
from novel_view_synthesis_3d_b200.diffusion import diffusion_tables
from novel_view_synthesis_3d_b200.srn_data import SRNScenes
from novel_view_synthesis_3d_b200.synthetic import _look_at
from tests import field_ref as F
from tests import lift_ref as LR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _orbit(V, up=(0.0, 0.0, 1.0), elev=(5.0, 55.0), r=1.3, seed=0):
    """V zero-roll look-at cameras at radius r with elevations in `elev` against up."""
    rng = np.random.RandomState(seed)
    up, e1, e2 = LR.band_basis(up)
    e = np.radians(rng.uniform(*elev, V))
    a = rng.uniform(0, 2 * np.pi, V)
    c = r * (np.sin(e)[:, None] * up + np.cos(e)[:, None] * (np.cos(a)[:, None] * e1 + np.sin(a)[:, None] * e2))
    return np.stack([LR.look_at(ci, up, e1) for ci in c]), c


# ---- 1. the draw ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('up,elev', [((0, 0, 1), (0.0, 60.0)), ((0.3, -1.0, 0.2), (-20.0, 35.0)), ((0, 1, 0), (-90.0, 90.0))])
def test_drawn_cameras_look_at_the_origin_inside_the_band(up, elev):
    P, r = 64, 1.7
    t, R, c = LR.draw(12, 3, P, 20, 980, up, elev, r)
    assert t.min() >= 20 and t.max() <= 980 and len(set(t.tolist())) > 40
    assert np.abs(R @ np.swapaxes(R, 1, 2) - np.eye(3)).max() < 1e-12
    assert np.abs(np.linalg.det(R) - 1).max() < 1e-12
    assert np.allclose(np.linalg.norm(c, axis=1), r, atol=1e-12)
    assert np.abs(R[:, :, 2] + c / r).max() < 1e-12                      # the optical axis points at the origin
    u = np.asarray(up, np.float64) / np.linalg.norm(up)
    assert np.abs(R[:, :, 0] @ u).max() < 1e-12                          # zero roll
    e = np.degrees(np.arcsin(c @ u / r))
    assert e.min() >= elev[0] - 1e-9 and e.max() <= elev[1] + 1e-9
    lo, hi = LI.elevation_range(c, up)
    assert lo == pytest.approx(e.min()) and hi == pytest.approx(e.max())
    assert not np.array_equal(LR.draw(12, 4, P, 20, 980, up, elev, r)[2], c)       # a new iteration draws afresh
    assert not np.array_equal(LR.draw(13, 3, P, 20, 980, up, elev, r)[2], c)


def test_z_up_is_synthetic_look_at():
    _, R, c = LR.draw(5, 1, 32, 0, 999, (0, 0, 1), (-80.0, 80.0), 1.3)
    up, e1, _ = LR.band_basis((0, 0, 1))
    assert np.array_equal(e1, [1.0, 0.0, 0.0])
    for Ri, ci in zip(R, c):
        assert np.array_equal(Ri, _look_at(ci))


def test_parallel_fallback():
    for up in ((0, 0, 1), (1, 2, -2)):
        _, R, c = LR.draw(1, 1, 4, 0, 999, up, (90.0, 90.0), 2.0)         # every draw at the pole: f parallel to up
        u, e1, _ = LR.band_basis(up)
        assert np.allclose(c, 2.0 * u, atol=1e-12)
        assert np.abs(R[:, :, 0] - e1).max() < 1e-15
        assert np.abs(R @ np.swapaxes(R, 1, 2) - np.eye(3)).max() < 1e-12 and np.abs(np.linalg.det(R) - 1).max() < 1e-12
        # near the pole, 0 < |f x up| < 1e-6: e1 is made perpendicular to f, so the camera stays orthonormal
        _, R, c = LR.draw(1, 1, 16, 0, 999, up, (89.99999, 90.0), 2.0)
        rn = np.linalg.norm(np.cross(-c / 2.0, u), axis=1)
        assert rn.max() < 1e-6 and rn.min() > 0.0
        assert np.abs(R @ np.swapaxes(R, 1, 2) - np.eye(3)).max() < 1e-14 and np.abs(np.linalg.det(R) - 1).max() < 1e-14
        assert np.abs(R[:, :, 2] + c / 2.0).max() < 1e-15
    assert np.array_equal(LR.look_at([0, 0, -1.3], np.array([0., 0, 1]), np.array([1., 0, 0])), _look_at(np.array([0, 0, -1.3])))


# ---- 2. estimate_up, elevation_range ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('up', [(0, 0, 1), (0.2, 0.9, -0.4)])
def test_estimate_up_recovers_the_up_of_look_at_cameras(up):
    R, c = _orbit(30, up=up)
    est, res = LI.estimate_up(R)
    u = np.asarray(up, np.float64) / np.linalg.norm(up)
    assert np.abs(est - u).max() < 1e-12 and res < 1e-12
    lo, hi = LI.elevation_range(c, est)
    assert 5.0 <= lo < hi <= 55.0


def test_estimate_up_of_rolled_cameras_has_a_large_residual():
    R, _ = _orbit(30)
    rolls = Rotation.from_rotvec(np.random.RandomState(1).uniform(-1.0, 1.0, 30)[:, None] * np.array([0, 0, 1.0])).as_matrix()
    _, res = LI.estimate_up(R @ rolls)                      # each camera rolled about its own optical axis
    assert res > 0.2


def test_estimate_up_of_srn_style_cameras():
    R = np.stack([_look_at(c) for c in np.random.RandomState(2).randn(20, 3) * [1, 1, 0.3] + [0, 0, 0.8]])
    up, res = LI.estimate_up(R)
    assert np.abs(up - [0, 0, 1]).max() < 1e-12 and res < 1e-12


# ---- 3. the residual ---------------------------------------------------------------------------------------------------------
def test_a_perfect_v_converts_to_the_true_eps():
    sa, sb = diffusion_tables()
    rng = np.random.RandomState(3)
    P, S = 3, 8
    t = np.array([20, 500, 980])
    x0 = rng.uniform(-1, 1, (P, S, S, 3))
    eps = rng.randn(P, S, S, 3)
    a, s = np.float64(sa)[t].reshape(P, 1, 1, 1), np.float64(sb)[t].reshape(P, 1, 1, 1)
    z = a * x0 + s * eps
    v = a * eps - s * x0
    for w in (0.0, 3.0):                                    # guidance of two equal outputs is the output itself
        got = LR.eps_hat(v, v, z, t, w, 'v', sa, sb)
        assert np.abs(got - eps).max() < 1e-5              # the fp32 tables: a^2 + s^2 = 1 to ~1e-7
        assert np.abs(LR.eps_hat(eps, eps, z, t, w, 'eps', sa, sb) - eps).max() < 1e-14


def test_image_grad_weights_and_clamp():
    sa, sb = diffusion_tables()
    P, S = 2, 4
    t = np.array([100, 900])
    rng = np.random.RandomState(4)
    out = rng.randn(2 * P, S, S, 3)
    out[0, 0, 0, 0] = np.inf
    out[1, 0, 0, 0] = 100.0
    eps = rng.randn(P, S, S, 3)
    render = rng.uniform(-1, 1, (P + 1, S, S, 3))
    x = rng.uniform(-1.2, 1.2, (S, S, 3))
    dC, sds, rec = LR.image_grad(out, None, eps, render, x, t, 2.0, 'eps', 1.5, 0.5, sa, sb)
    r = 3.0 * out[:P] - 2.0 * out[P:] - eps
    r = np.clip(np.where(np.isfinite(r), r, 0), -16, 16)
    assert r[0, 0, 0, 0] == 0 and r[1, 0, 0, 0] == 16
    om = np.float64(sb)[t] ** 2
    assert np.allclose(dC[:P], 2 * 1.5 * om[:, None, None, None] * r / (3 * S * S * P))
    d = (render[P] + 1) / 2 - np.clip((x + 1) / 2, 0, 1)
    assert np.allclose(dC[P], 2 * 0.5 * d / (3 * S * S))
    assert sds == pytest.approx(np.mean(r ** 2)) and rec == pytest.approx(np.mean(d ** 2))


# ---- 4. the render backward ------------------------------------------------------------------------------------------------
def test_render_backward_matches_central_differences():
    G, S, V = 5, 4, 2
    R, c = _orbit(V, seed=5)
    f = 131.25 * S / 128
    K = np.tile(np.array([[f, 0, S / 2], [0, f, S / 2], [0, 0, 1.0]]), (V, 1, 1))
    b = 0.95 * 1.3 / math.sqrt(3)
    step = b / (G - 1)
    rng = np.random.RandomState(6)
    grid = rng.randn(G, G, G, 4) * 2 + np.array([8.0, 0, 0, 0])
    dC = rng.uniform(-1.9, 1.9, (V, S, S, 3))
    g = LR.render_backward(grid, dC, R, c, K, b, 0.0, step, 0.3, tv=(0.01, 0.02)).numpy()

    def f_(gr):
        gt = torch.as_tensor(gr)
        C = (F.render(gt, R, c, K, S, b, 0.0, step, 0.3) + 1) / 2
        return float((C * torch.as_tensor(dC)).sum() + F.tv(gt, 0.01, 0.02))

    idx = [tuple(rng.randint(0, G, 3)) + (q,) for q in range(4) for _ in range(6)]
    h = 1e-5
    for i in idx:
        e = np.zeros_like(grid)
        e[i] = h
        fd = (f_(grid + e) - f_(grid - e)) / (2 * h)
        assert abs(fd - g[i]) <= 1e-6 + 1e-5 * abs(g[i]), (i, fd, g[i])
    assert np.abs(g).max() > 1e-3


def test_render_backward_reads_non_finite_as_zero_and_applies_the_unit():
    G, S = 4, 3
    R, c = _orbit(1, seed=7)
    K = np.array([[[3.0, 0, 1.5], [0, 3.0, 1.5], [0, 0, 1]]])
    grid = np.random.RandomState(8).randn(G, G, G, 4)
    dC = np.random.RandomState(9).randn(1, S, S, 3) * 5
    dC[0, 0, 0, 0] = np.nan
    kw = dict(bound=0.7, near=0.0, step=0.1, background=1.0)
    a = LR.render_backward(grid, dC, R, c, K, unit=2.0 ** -10, **kw)
    b = LR.render_backward(grid, np.nan_to_num(dC, nan=0.0) * 2.0 ** -10, R, c, K, **kw)
    assert torch.equal(a, b)


def test_grad_unit():
    for sw, rw in ((1.0, 1.0), (2.0, 0.5), (0.0, 3.0), (1e-3, 0.0), (250.0, 7.0)):
        u = LI.grad_unit(sw, rw)
        assert u == LR.grad_unit(sw, rw) and math.log2(u) == int(math.log2(u))
        l1 = 32 * sw + 2 * rw
        assert LI.MAX_GRAD_L1 / 2 < l1 / u <= LI.MAX_GRAD_L1      # the smallest power of two within the bound
    assert LI.grad_unit(0.0, 0.0) == 1.0
    # at S = 128, P = 2 the default weights give values of order 1 (2 omega r / (3 S^2 P) / u), not ~7e-6
    assert 1.0 < 2.0 / (3 * 128 * 128 * 2) / LI.grad_unit(1.0, 1.0) < 4.0


# ---- 5. constants, errors ----------------------------------------------------------------------------------------------------
def test_header_constants():
    hdr = open(os.path.join(ROOT, 'include', 'xunet_b200.h')).read()
    d = dict(re.findall(r'#define (XUNET_(?:LIFT|FIELD)_\w+) (\S+)', hdr))
    assert int(d['XUNET_LIFT_SEED_DOMAIN'].rstrip('ULL'), 16) == LI.SEED_DOMAIN == LR.SEED_DOMAIN
    assert float(d['XUNET_LIFT_MAX_RESIDUAL'].rstrip('f')) == LI.MAX_RESIDUAL == LR.MAX_RESIDUAL
    assert float(d['XUNET_FIELD_MAX_GRAD_L1']) == LI.MAX_GRAD_L1 == 2.0 ** 23
    assert LI.MAX_PIXELS == 1 << 20


def test_constructor_errors_before_any_device_work():
    for kw, what in ((dict(w=None), 'w=None'), (dict(w=-1.0), 'w'), (dict(w=float('nan')), 'w'), (dict(draws=0), 'draws'),
                     (dict(t_range=(10, 1000)), 't_range'), (dict(t_range=(7, 3)), 't_range'), (dict(grid=1), 'grid'),
                     (dict(grid=257), 'grid')):
        with pytest.raises(ValueError, match=what):
            LI.FieldLifter(None, None, 16, **kw)
    with pytest.raises(ValueError, match='pixels'):
        LI.FieldLifter(None, None, 256, draws=16)


# ---- 6. examples/lift_srn.py -------------------------------------------------------------------------------------------------
def _example():
    spec = importlib.util.spec_from_file_location('lift_srn', os.path.join(ROOT, 'examples', 'lift_srn.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_example_helpers_on_a_synthetic_scene(tmp_path):
    ex = _example()
    a = ex.parse_args([str(tmp_path), '--ckpt', 'c', '--side', '16', '--targets', '3', '--draws', '3', '--grid', '24',
                       '--prediction', 'v', '--ray-convention', 'opencv_uv', '--save-renders'])
    assert a.side == 16 and a.targets == 3 and a.draws == 3 and a.grid == 24 and a.prediction == 'v' and a.save_renders
    assert a.source_view == 64 and a.iters == LI.ITERS and a.w == LI.W
    with pytest.raises(SystemExit):
        ex.parse_args([str(tmp_path), '--draws', '0'])
    # a scene directory in SRN's layout: two instances of 7 views on the upper half of a sphere of radius 1.3
    R, c = _orbit(14, elev=(10.0, 50.0), seed=11)
    rng = np.random.RandomState(12)
    for i in range(2):
        d = tmp_path / f'obj{i}'
        (d / 'rgb').mkdir(parents=True)
        (d / 'pose').mkdir()
        (d / 'intrinsics.txt').write_text('131.25 64.0 64.0 0.\n0. 0. 0.\n1.\n128 128\n')
        for v in range(7):
            cv2.imwrite(str(d / 'rgb' / f'{v:06d}.png'), rng.randint(0, 256, (32, 32, 3), dtype=np.uint8))
            pose = np.eye(4)
            pose[:3, :3], pose[:3, 3] = R[7 * i + v], c[7 * i + v]
            (d / 'pose' / f'{v:06d}.txt').write_text(' '.join(f'{x:.9f}' for x in pose.reshape(-1)) + '\n')
    ds = SRNScenes(str(tmp_path), img_sidelength=16)
    d = ds.instance_views(1)
    assert ex.select_targets(7, 4, 3) == [0, 2, 5]
    up, res, elev = ex.camera_band(d['R'], d['t'])
    assert np.abs(up - [0, 0, 1]).max() < 1e-6 and res < 1e-6          # the poses are stored to 9 decimals
    want = LI.elevation_range(d['t'], up)
    assert elev == pytest.approx(want) and 10.0 <= elev[0] <= elev[1] <= 50.0
    recs = [dict(instance='a', view=0, psnr=20.0, ssim=0.5), dict(instance='a', view=1, psnr=30.0, ssim=0.7)]
    s = ex.summarize(recs)
    assert s['n_views'] == 2 and s['mean_psnr'] == pytest.approx(25.0) and s['mean_ssim'] == pytest.approx(0.6)
    assert ex.summarize([])['n_views'] == 0
