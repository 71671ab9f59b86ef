"""Image metrics without a GPU: the float64 SSIM reference against an independent explicit-window implementation and known
answers, SRNScenes.instance_views, and the target selection of examples/eval_srn.py."""
import importlib.util
import os

import numpy as np
import pytest

from tests import ssim_ref as M

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ssim_window(pred, target) -> np.ndarray:
    """Second float64 SSIM: the 11x11 Gaussian window applied explicitly at every interior pixel (no scipy)."""
    i = np.arange(-5, 6)
    g = np.exp(-i * i / (2 * 1.5 ** 2))
    g /= g.sum()
    w2 = np.outer(g, g)
    up, ut = M.to_unit(pred), M.to_unit(target)
    out = []
    for p_img, t_img in zip(up, ut):
        s = []
        for c in range(3):
            p, t = p_img[..., c], t_img[..., c]
            win = lambda a: np.einsum('ijkl,kl->ij', np.lib.stride_tricks.sliding_window_view(a, (11, 11)), w2)
            s.append(M.ssim_from_moments(win(p), win(t), win(p * p), win(t * t), win(p * t)))
        out.append(np.mean(s))
    return np.asarray(out)


@pytest.mark.parametrize('S', [11, 16, 64])
@pytest.mark.parametrize('kind', ['noise', 'smooth', 'srn'])
def test_reference_matches_explicit_window(kind, S):
    p, t = M.make_pair(kind, 2, S, seed=S)
    a, b = M.ssim(p, t), ssim_window(p, t)
    assert a.shape == (2,) and np.all(np.abs(a - b) <= 1e-12), (a, b)
    assert np.all(np.abs(a) <= 1)


def test_identical_images():
    p, _ = M.make_pair('noise', 2, 16)
    mse, psnr = M.mse_psnr(p, p)
    assert np.all(mse == 0) and np.all(np.isposinf(psnr))
    assert np.allclose(M.ssim(p, p), 1.0, rtol=0, atol=1e-12)
    assert np.allclose(ssim_window(p, p), 1.0, rtol=0, atol=1e-12)


@pytest.mark.parametrize('va,vb', [(0.5, -0.25), (-1.0, 1.0), (0.9, 0.8)])
def test_constant_images_pin_c1_and_the_range_map(va, vb):
    S = 16
    p, t = np.full((1, S, S, 3), va, np.float32), np.full((1, S, S, 3), vb, np.float32)
    a, b = (np.float64(np.float32(va)) + 1) / 2, (np.float64(np.float32(vb)) + 1) / 2
    want = (2 * a * b + M.C1) / (a * a + b * b + M.C1)
    assert np.isclose(M.ssim(p, t)[0], want, rtol=0, atol=1e-10)
    assert np.isclose(ssim_window(p, t)[0], want, rtol=0, atol=1e-10)
    assert np.isclose(M.mse_psnr(p, t)[0][0], (a - b) ** 2, rtol=1e-12, atol=0)


def test_offset_of_a_tenth_is_20_db():
    rng = np.random.RandomState(3)
    t = rng.uniform(-0.9, 0.7, (2, 16, 16, 3))
    p = t + 0.2                                         # u_pred = u_target + 0.1, nothing clipped
    mse, psnr = M.mse_psnr(p, t)
    assert np.allclose(mse, 0.01, rtol=1e-9) and np.allclose(psnr, 20.0, rtol=0, atol=1e-8)


def test_out_of_range_inputs_score_as_clamped():
    rng = np.random.RandomState(4)
    p, t = 1.5 * rng.uniform(-1, 1, (2, 16, 16, 3)), 1.5 * rng.uniform(-1, 1, (2, 16, 16, 3))
    pc, tc = np.clip(p, -1, 1), np.clip(t, -1, 1)
    assert np.array_equal(M.ssim(p, t), M.ssim(pc, tc))
    assert np.array_equal(M.mse_psnr(p, t)[0], M.mse_psnr(pc, tc)[0])


# ---- SRNScenes.instance_views -------------------------------------------------------------------------------------------
def test_instance_views_shapes_order_and_values(tmp_path):
    pytest.importorskip('cv2')
    from tests.test_srn_data import _make_tree
    from novel_view_synthesis_3d_b200 import srn_data as D
    _make_tree(str(tmp_path), n_inst=2, n_views=5, H=32, W=32)
    ds = D.SRNScenes(str(tmp_path), img_sidelength=16)
    d = ds.instance_views(1)
    assert d['name'] == 'obj1'
    assert d['x'].shape == (5, 16, 16, 3) and d['R'].shape == (5, 3, 3) and d['t'].shape == (5, 3) and d['K'].shape == (3, 3)
    assert np.array_equal(d['t'][:, 1], np.arange(5))                     # pose t = [instance, view, 1.3]: sorted file order
    for j in range(5):
        assert np.array_equal(d['x'][j], D.load_rgb(str(tmp_path / 'obj1' / 'rgb' / f'{j:06d}.png'), 16))
        pose = D.load_pose(str(tmp_path / 'obj1' / 'pose' / f'{j:06d}.txt'))
        assert np.array_equal(d['R'][j], pose[:3, :3]) and np.array_equal(d['t'][j], pose[:3, 3])
    assert np.array_equal(d['K'], ds.instances[1]['K'])
    sub = D.SRNScenes(str(tmp_path), img_sidelength=16, max_observations_per_instance=3).instance_views(0)
    assert np.array_equal(sub['t'][:, 1], [0, 1, 3])                      # the reader's evenly spaced subset


def test_instance_views_leaves_the_batch_stream_alone(tmp_path):
    pytest.importorskip('cv2')
    from tests.test_srn_data import _make_tree
    from novel_view_synthesis_3d_b200 import srn_data as D
    _make_tree(str(tmp_path), n_inst=2, n_views=4, H=32, W=32)
    a = D.SRNScenes(str(tmp_path), img_sidelength=16, host_diffusion=True, seed=5)
    b = D.SRNScenes(str(tmp_path), img_sidelength=16, host_diffusion=True, seed=5)
    b.instance_views(0)
    b.instance_views(1)
    ia, ib = a.batches(3), b.batches(3)
    for _ in range(3):
        x, y = next(ia), next(ib)
        assert x.keys() == y.keys() and all(np.array_equal(x[k], y[k]) for k in x)


# ---- target selection of examples/eval_srn.py ---------------------------------------------------------------------------
def _eval_script():
    spec = importlib.util.spec_from_file_location('eval_srn', os.path.join(REPO, 'examples', 'eval_srn.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_select_targets():
    sel = _eval_script().select_targets
    rest = [v for v in range(251) if v != 64]
    t = sel(251, 64, 10)
    assert len(t) == 10 and 64 not in t and t == sorted(t)
    assert t == [rest[i] for i in range(0, 250, 25)]                       # every 25th of the 250 other views
    assert sel(251, 64, 0) == rest and sel(251, 64, 250) == rest and sel(251, 64, 1000) == rest
    assert sel(6, 2, 2) == [0, 3] and sel(6, 5, 0) == [0, 1, 2, 3, 4]
    gaps = np.diff([rest.index(v) for v in sel(251, 64, 7)])
    assert gaps.max() - gaps.min() <= 1                                     # evenly spaced over the remaining views
