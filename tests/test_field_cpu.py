"""CPU checks of the float64 reference of the radiance grid (tests/field_ref.py) that the GPU tests compare the kernels against:
its rays, its background, a homogeneous cube against the closed form, its gradient against finite differences, and the
constants it shares with include/xunet_b200.h and novel_view_synthesis_3d_b200.consistency."""
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import xunet_ref as O
from novel_view_synthesis_3d_b200 import consistency as CS
from novel_view_synthesis_3d_b200.synthetic import _look_at
from tests import field_ref as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cameras(V, S, seed=0, r=1.3):
    rng = np.random.RandomState(seed)
    c = rng.randn(V, 3)
    c = r * c / np.linalg.norm(c, axis=1, keepdims=True)
    R = np.stack([_look_at(x) for x in c])
    f = 131.25 * S / 128.
    K = np.tile(np.array([[f, 0, S / 2.], [0, f, S / 2.], [0, 0, 1.]])[None], (V, 1, 1))
    return R, c, K


def test_rays_are_the_oracles_opencv_uv_rays():
    R, t, K = cameras(3, 16)
    K[1, 0, 1] = 0.7                       # a skewed camera too
    o, d = F.rays(R, t, K, 16)
    po, pd = O.camera_rays(*(torch.as_tensor(x, dtype=torch.float64) for x in (R, t, K)), 16, 16, convention='opencv_uv')
    assert torch.allclose(o, po, rtol=0, atol=1e-14) and torch.allclose(d, pd, rtol=0, atol=1e-14)


def test_empty_space_and_missed_rays_render_the_background():
    G, S, b = 8, 12, 0.7
    R, t, K = cameras(2, S)
    grid = torch.zeros(G, G, G, 4, dtype=torch.float64)
    grid[..., 0] = -1e4
    grid[..., 1:] = torch.randn(G, G, G, 3, dtype=torch.float64)
    img = F.render(grid, R, t, K, S, b, 0.0, b / (G - 1), -0.3)
    assert torch.all(img == -0.3) or torch.allclose(img, torch.full_like(img, -0.3), rtol=0, atol=1e-15)
    # a camera looking away from the cube, and one whose rays pass beside it: every ray misses
    o = torch.tensor([[0., 0., 2.], [2., 2., 0.]], dtype=torch.float64)
    d = torch.tensor([[0., 0., 1.], [0., 0., 1.]], dtype=torch.float64)
    grid[..., 0] = 50.0
    C = F.composite(grid, o, d, b, 0.0, b / (G - 1), 0.5)
    assert torch.all(C == 0.75)


@pytest.mark.parametrize('near', [0.0, 1.2])
def test_homogeneous_cube_is_the_closed_form(near):
    G, b, step = 5, 0.6, 0.07
    raw0, rawc = 1.3, torch.tensor([0.4, -1.1, 2.0], dtype=torch.float64)
    grid = torch.empty(G, G, G, 4, dtype=torch.float64)
    grid[..., 0] = raw0
    grid[..., 1:] = rawc
    sigma = math.log1p(math.exp(raw0 + F.DENSITY_SHIFT))
    c = torch.sigmoid(rawc)
    s3 = 1 / math.sqrt(3)
    # origin, direction, where the ray enters the cube and its chord (an axis through the centre, the main diagonal, and a
    # ray parallel to an axis off-centre, whose other two direction components are zero)
    cases = [((0., 0., -1.), (0., 0., 1.), 1 - b, 2 * b), ((-1., -1., -1.), (s3, s3, s3), math.sqrt(3) * (1 - b), 2 * b * math.sqrt(3)),
             ((0.2, -0.3, -2.), (0., 0., 1.), 2 - b, 2 * b)]
    for o, d, enter, chord in cases:
        o, d = torch.tensor([o], dtype=torch.float64), torch.tensor([d], dtype=torch.float64)
        Lx = enter + chord - max(enter, near)          # the part past near
        _, L, _ = F.segments(o, d, b, near)
        assert abs(float(L[0]) - Lx) <= 1e-12
        C = F.composite(grid, o, d, b, near, step, 0.2)[0]
        T = math.exp(-sigma * Lx)
        want = c * (1 - T) + 0.6 * T
        assert torch.allclose(C, want, rtol=0, atol=1e-12), (o, C, want)


def test_gradient_matches_finite_differences():
    G, S, b = 6, 8, 0.7
    R, t, K = cameras(2, S, seed=3)
    rng = np.random.RandomState(1)
    grid = torch.as_tensor(rng.randn(G, G, G, 4) * np.array([3.0, 1.0, 1.0, 1.0]) + np.array([4.0, 0, 0, 0]),
                           dtype=torch.float64).requires_grad_(True)
    views = rng.uniform(-1, 1, (2, S, S, 3))
    pix = CS.draw_rays(5, 1, 64, 2 * S * S)
    step = b / (G - 1)

    def f(g):
        return F.data_loss(g, views, R, t, K, pix, b, 0.0, step, 1.0) + F.tv(g, 0.3, 0.05)

    (gr,) = torch.autograd.grad(f(grid), grid)
    with torch.no_grad():
        flat = grid.detach().reshape(-1)
        pick = rng.choice(flat.numel(), 60, replace=False)
        pick = np.concatenate([pick, np.argsort(-gr.abs().reshape(-1).numpy())[:20]])
        h = 1e-5
        for j in pick:
            e = torch.zeros_like(flat)
            e[j] = h
            fd = (f((flat + e).reshape(grid.shape)) - f((flat - e).reshape(grid.shape))) / (2 * h)
            assert abs(float(fd) - float(gr.reshape(-1)[j])) <= 1e-7 * max(1.0, float(gr.abs().max())), (j, float(fd))
    assert float(gr.abs().max()) > 1e-3     # the check is not vacuous


def _defines():
    hdr = open(os.path.join(ROOT, 'include', 'xunet_b200.h')).read()
    return {k: v for k, v in re.findall(r'#define (XUNET_FIELD_\w+) \(?([^)/\n]+?)f?\)?\s*(?:/\*.*)?$', hdr, re.M)}


def test_header_constants_are_the_references():
    d = _defines()
    assert float(d['XUNET_FIELD_DENSITY_SHIFT']) == F.DENSITY_SHIFT == CS.DENSITY_SHIFT
    assert int(d['XUNET_FIELD_MIN_GRID']) == F.MIN_GRID == CS.MIN_GRID
    assert int(d['XUNET_FIELD_MAX_GRID']) == F.MAX_GRID == CS.MAX_GRID
    assert float(d['XUNET_FIELD_MAX_BOUND']) == F.MAX_BOUND == CS.MAX_BOUND
    assert int(d['XUNET_FIELD_MAX_SAMPLES']) == F.MAX_SAMPLES == CS.MAX_SAMPLES
    assert eval(d['XUNET_FIELD_MAX_RAYS']) == F.MAX_RAYS == CS.MAX_RAYS
    assert float(d['XUNET_FIELD_FIXED_ONE']) == F.FIXED_ONE == CS.FIXED_ONE
    # an all-zero grid is nearly transparent: along the longest chord of the default cube of SRN's r = 1.3 cameras
    b = CS.default_bound(np.array([[0, 0, 1.3]]))
    assert math.exp(-math.log1p(math.exp(F.DENSITY_SHIFT)) * 2 * math.sqrt(3) * b) > 0.99


def test_ray_draw_restates_the_hash():
    pix = CS.draw_rays(7, 3, 5, 1000)
    m = (1 << 64) - 1

    def mix(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
        return z ^ (z >> 31)
    want = [mix((7 * 0x9E3779B97F4A7C15 + 3 * 0xD1B54A32D192ED03 + r) & m) % 1000 for r in range(5)]
    assert pix.tolist() == want


def test_held_out_split():
    assert CS.held_out(17, 8) == [7, 15]
    assert CS.held_out(3, 2) == [1]
