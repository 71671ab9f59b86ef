"""The radiance grid of the 3D consistency score on the device (xunet_field_render, xunet_field_loss_grad, consistency.py):
render, loss and gradient parity with the float64 reference of tests/field_ref.py, determinism, recovery of an analytic scene,
discrimination of an inconsistent view set, argument checks, and examples/consistency_srn.py end to end."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib, consistency as CS
from tests import field_ref as F
from tests.test_field_cpu import cameras

pytestmark = pytest.mark.gpu


def _bits(x):
    return x.detach().cpu().numpy().view(np.uint32).copy()


def smooth_grid(G, seed, density=12.0):
    """Raw values made of a few low-frequency sinusoids: density from empty to nearly opaque along a chord, colour in +-2."""
    rng = np.random.RandomState(seed)
    x = np.linspace(-1, 1, G)
    X = np.stack(np.meshgrid(x, x, x, indexing='ij'), -1)
    g = np.zeros((G, G, G, 4))
    for c in range(4):
        for _ in range(3):
            k, ph = rng.uniform(-3, 3, 3), rng.uniform(0, 2 * np.pi)
            g[..., c] += np.sin(X @ k + ph)
    g[..., 0] = density * g[..., 0] / 3 + density / 2
    return g


def cameras_with_miss(V, S, seed=0):
    """synthetic.py's cameras on the r = 1.3 sphere, plus one close to the cube looking past its corner (part of its rays miss)."""
    R, t, K = cameras(V - 1, S, seed=seed)
    from novel_view_synthesis_3d_b200.synthetic import _look_at
    c = np.array([0.2, -0.1, 1.1])
    Rm = _look_at(c - np.array([0.9, 0.9, 0.0]))
    return np.concatenate([R, Rm[None]]), np.concatenate([t, c[None]]), np.concatenate([K, K[:1]])


def _render(grid, R, t, K, S, b, step, near=0.0, background=1.0):
    f = CS.Field(grid=torch.as_tensor(grid, dtype=torch.float32).cuda().contiguous(), bound=b, step=step, near=near,
                 background=background, S=S, loss=None)
    return f.render(R, t, K)


# ---- 1. render parity -------------------------------------------------------------------------------------------------------
# fp32 against fp64: a pixel composites at most 2 sqrt(3) (G - 1) ~ 220 samples (G = 64), each adding O(6e-8) relative rounding to
# T and C, so |C - C_ref| stays near 220 * 6e-8 ~ 1.3e-5 even if every rounding lined up; sample positions carry ~ G |t| 6e-8 ~ 1e-5
# grid units of error into raw values that change O(1) per unit.  The pixel 2C - 1 doubles it: 1e-4 keeps a 3x margin.
@pytest.mark.parametrize('G', [17, 64])
@pytest.mark.parametrize('S', [16, 64])
def test_render_matches_reference(G, S):
    R, t, K = cameras_with_miss(4, S, seed=G + S)
    b = CS.default_bound(t[:-1])
    step = b / (G - 1)
    g = smooth_grid(G, seed=G)
    got = _render(g, R, t, K, S, b, step, near=0.05, background=0.4).double().cpu()
    want = F.render(torch.as_tensor(g), R, t, K, S, b, 0.05, step, 0.4)
    miss = (got[-1] - 0.4).abs() <= 1e-6
    assert miss.any() and not miss.all()       # the last camera's rays partly miss the cube
    err = (got - want).abs().max().item()
    assert err <= 1e-4, err


# ---- 2. loss and gradient parity --------------------------------------------------------------------------------------------
def _loss_grad(lib, g, views, R, t, K, b, step, rays, seed, it, tv=(0.02, 0.01), background=1.0):
    G, V, S = g.shape[0], views.shape[0], views.shape[1]
    dev = torch.device('cuda')
    gd = torch.as_tensor(g, dtype=torch.float32, device=dev).contiguous()
    vd = torch.as_tensor(views, dtype=torch.float32, device=dev).contiguous()
    Rd, td, Kd = (torch.as_tensor(x, dtype=torch.float32, device=dev).contiguous() for x in (R, t, K))
    kinv = torch.empty(V, 9, device=dev)
    acc = torch.zeros(4 * G ** 3 + 1, dtype=torch.int64, device=dev)
    grad = torch.empty_like(gd)
    loss = torch.full((it,), -1.0, device=dev)
    count = torch.full((1,), it, dtype=torch.int64, device=dev)
    _lib.check(lib.xunet_field_loss_grad(gd.data_ptr(), G, b, vd.data_ptr(), Rd.data_ptr(), td.data_ptr(), Kd.data_ptr(),
                                         kinv.data_ptr(), V, S, 0.0, step, background, rays, count.data_ptr(), seed, tv[0], tv[1],
                                         acc.data_ptr(), grad.data_ptr(), loss.data_ptr(), it, torch.cuda.current_stream().cuda_stream),
               'loss_grad')
    torch.cuda.synchronize()
    assert int(acc.abs().max()) == 0          # the call hands the fixed-point buffer back cleared
    return loss, grad


# Loss: each ray's C carries <= ~55 samples of fp32 rounding (G = 17), ~3e-6 absolute at worst, against |C - u| ~ 0.3 for these
# unrelated targets, and the fixed-point quantum 2^-33 per ray is 1e-8 of a squared error ~0.1: 1e-5 relative bounds both.
# Gradient: each word sums fp32 per-sample products (~1e-6 relative each) and at most rays * 55 roundings of 2^-33 / 3N; 1e-4 of
# max |g| leaves two orders of magnitude.
def test_loss_and_gradient_match_autograd(lib):
    G, S, V, rays, seed, it = 17, 16, 3, 4096, 11, 3
    R, t, K = cameras_with_miss(V, S, seed=5)
    b = CS.default_bound(t[:-1])
    step = b / (G - 1)
    g = smooth_grid(G, seed=2)
    views = np.random.RandomState(3).uniform(-1, 1, (V, S, S, 3))
    loss, grad = _loss_grad(lib, g, views, R, t, K, b, step, rays, seed, it)
    assert loss[:it - 1].eq(-1).all()        # only loss_out[i - 1] is written
    gt = torch.as_tensor(g).requires_grad_(True)
    pix = CS.draw_rays(seed, it, rays, V * S * S)
    data = F.data_loss(gt, views, R, t, K, pix, b, 0.0, step, 1.0)
    (want,) = torch.autograd.grad(data + F.tv(gt, 0.02, 0.01), gt)
    assert abs(loss[it - 1].item() - data.item()) <= 1e-5 * data.item(), (loss[it - 1].item(), data.item())
    err = (grad.double().cpu() - want).abs().max().item()
    assert err <= 1e-4 * want.abs().max().item(), (err, want.abs().max().item())


# ---- 3. determinism ---------------------------------------------------------------------------------------------------------
def _scene_views(n=12, S=32, seed=0):
    R, t, K = cameras(n, S, seed=seed)
    b = CS.default_bound(t)
    G = 32
    v = _render(sphere_grid(G, b, SPHERES), R, t, K, S, b, b / (G - 1))
    return v, R, t, K


def test_fits_are_bit_identical_and_graph_replay_equals_eager():
    v, R, t, K = _scene_views()
    kw = dict(iters=50, rays=2048, seed=4)
    a = CS.fit_field(v, R, t, K, **kw)
    b = CS.fit_field(v, R, t, K, **kw)
    c = CS.fit_field(v, R, t, K, use_graph=False, **kw)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(a.grid), _bits(b.grid)) and np.array_equal(_bits(a.grid), _bits(c.grid))
    assert np.array_equal(_bits(a.loss), _bits(b.loss)) and np.array_equal(_bits(a.loss), _bits(c.loss))
    assert a.loss[-1].item() < a.loss[0].item()
    assert not np.array_equal(_bits(a.grid), _bits(CS.fit_field(v, R, t, K, iters=50, rays=2048, seed=5).grid))


def test_a_view_renders_the_same_alone_and_in_a_batch():
    v, R, t, K = _scene_views()
    f = CS.fit_field(v, R, t, K, iters=20, rays=2048)
    full = _bits(f.render(R, t, K))
    for i in (0, 5, 11):
        assert np.array_equal(_bits(f.render(R[i:i + 1], t[i:i + 1], K[i:i + 1]))[0], full[i])


# ---- 4./5. recovery of a consistent scene, discrimination of an inconsistent one -----------------------------------------------
SPHERES = [((0.22, 0.0, 0.05), 0.2, (0.9, 0.2, 0.15)), ((-0.2, 0.18, 0.1), 0.16, (0.15, 0.7, 0.25)),
           ((0.0, -0.22, -0.15), 0.18, (0.2, 0.3, 0.9)), ((0.05, 0.12, -0.25), 0.12, (0.95, 0.85, 0.2))]


def sphere_grid(G, b, spheres, offsets=None):
    """Soft coloured spheres sampled into a (G, G, G, 4) raw grid: raw density 60 inside, fading over 0.02 at the surface."""
    x = torch.linspace(-b, b, G, dtype=torch.float64, device='cuda')
    X = torch.stack(torch.meshgrid(x, x, x, indexing='ij'), -1)
    occ, num = [], 0
    for j, (c, r, col) in enumerate(spheres):
        c = torch.tensor(c, dtype=torch.float64, device='cuda') + (0 if offsets is None else torch.as_tensor(offsets[j]).cuda())
        o = torch.sigmoid((r - torch.linalg.norm(X - c, dim=-1)) / 0.02)
        occ.append(o)
        num = num + o[..., None] * torch.logit(torch.tensor(col, dtype=torch.float64, device='cuda'))
    occ_t = torch.stack(occ)
    g = torch.empty(G, G, G, 4, dtype=torch.float64, device='cuda')
    g[..., 0] = 60 * occ_t.max(0).values
    g[..., 1:] = num / (occ_t.sum(0)[..., None] + 1e-6)
    return g.float()


def _scene_sets(S=64, G=64, V=48, shift=0.04, seed=0):
    R, t, K = cameras(V, S, seed=seed)
    b = CS.default_bound(t)
    step = b / (G - 1)
    good = _render(sphere_grid(G, b, SPHERES), R, t, K, S, b, step)
    rng = np.random.RandomState(seed + 1)
    bad = torch.cat([_render(sphere_grid(G, b, SPHERES, rng.randn(len(SPHERES), 3) * shift * b), R[i:i + 1], t[i:i + 1], K[i:i + 1],
                             S, b, step) for i in range(V)])
    return good, bad, R, t, K


# Measured with the fit_field defaults on an H100 80GB HBM3 (the fit is deterministic, so every run gives these bits): the
# consistent set scores 43.75 dB / SSIM 0.9926 on its 8 held-out views, the inconsistent one 18.29 dB / 0.6306 (25.46 dB lower).
RECOVERY_FLOOR_DB = 40.0
MARGIN_DB = 20.0


def test_consistent_views_are_recovered_and_inconsistent_ones_score_lower():
    good, bad, R, t, K = _scene_sets()
    sg = CS.consistency_score(good, R, t, K, every=6)
    sb = CS.consistency_score(bad, R, t, K, every=6)
    print(f'consistency: consistent {sg["mean_psnr"]:.2f} dB / {sg["mean_ssim"]:.4f}, inconsistent {sb["mean_psnr"]:.2f} dB / '
          f'{sb["mean_ssim"]:.4f}, fit losses {sg["fit_loss"]:.2e} / {sb["fit_loss"]:.2e}')
    assert len(sg['held_out']) == 8 and sg['held_out'] == [5, 11, 17, 23, 29, 35, 41, 47]
    assert all(math.isfinite(x) for x in sg['psnr'] + sb['psnr'] + sg['ssim'] + sb['ssim'])
    assert sg['mean_psnr'] >= RECOVERY_FLOOR_DB, sg
    assert sg['mean_psnr'] - sb['mean_psnr'] >= MARGIN_DB, (sg['mean_psnr'], sb['mean_psnr'])


# ---- 6. argument errors -----------------------------------------------------------------------------------------------------
def test_c_abi_rejects_bad_arguments(lib):
    G, S, V = 8, 8, 2
    R, t, K = (torch.as_tensor(x, dtype=torch.float32).cuda().contiguous() for x in cameras(V, S))
    g = torch.zeros(G, G, G, 4, device='cuda')
    views = torch.zeros(V, S, S, 3, device='cuda')
    kinv = torch.full((V, 9), 7.0, device='cuda')
    out = torch.full((V, S, S, 3), 7.0, device='cuda')
    acc = torch.zeros(4 * G ** 3 + 1, dtype=torch.int64, device='cuda')
    grad = torch.full_like(g, 7.0)
    loss = torch.full((4,), 7.0, device='cuda')
    count = torch.ones(1, dtype=torch.int64, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    p = {k: x.data_ptr() for k, x in dict(g=g, R=R, t=t, K=K, kinv=kinv, out=out, views=views, acc=acc, grad=grad, loss=loss,
                                           count=count).items()}
    good_r = dict(grid=p['g'], G=G, bound=0.7, R=p['R'], t=p['t'], K=p['K'], kinv=p['kinv'], V=V, S=S, near=0.0, step=0.1,
                  background=1.0, out=p['out'])
    good_l = dict(grid=p['g'], G=G, bound=0.7, views=p['views'], R=p['R'], t=p['t'], K=p['K'], kinv=p['kinv'], V=V, S=S, near=0.0,
                  step=0.1, background=1.0, rays=64, iter_dev=p['count'], seed=0, tv_d=0.0, tv_c=0.0, acc=p['acc'],
                  grad=p['grad'], loss=p['loss'], loss_len=4)
    shared = [dict(G=1), dict(G=257), dict(S=0), dict(V=0), dict(bound=0.0), dict(bound=-1.0), dict(bound=float('nan')),
              dict(bound=65.0), dict(step=0.0), dict(step=float('inf')), dict(near=-0.1), dict(near=float('nan')),
              dict(step=1e-4), dict(background=float('nan'))]
    cases_r = shared + [{k: None} for k in ('grid', 'R', 't', 'K', 'kinv', 'out')]
    cases_l = shared + [{k: None} for k in ('grid', 'views', 'R', 't', 'K', 'kinv', 'iter_dev', 'acc', 'grad', 'loss')] + \
        [dict(rays=0), dict(rays=(1 << 20) + 1), dict(tv_d=-1.0), dict(tv_c=float('nan')), dict(loss_len=-1)]
    for fn, good, cases in ((lib.xunet_field_render, good_r, cases_r), (lib.xunet_field_loss_grad, good_l, cases_l)):
        for bad in cases:
            args = dict(good, **bad)
            assert fn(*args.values(), st) != 0, (fn.__name__, bad)
            assert lib.xunet_last_error().decode().startswith(fn.__name__), (fn.__name__, bad)
    torch.cuda.synchronize()
    for x in (kinv, out, grad, loss):                  # nothing was launched
        assert x.eq(7.0).all()
    assert acc.eq(0).all()
    assert lib.xunet_field_render(*good_r.values(), st) == 0
    assert lib.xunet_field_loss_grad(*good_l.values(), st) == 0
    torch.cuda.synchronize()
    assert not out.eq(7.0).any() and not grad.eq(7.0).any() and loss[0].item() != 7.0


def test_python_rejects_bad_inputs():
    v = np.zeros((3, 16, 16, 3), np.float32)
    R, t, K = cameras(3, 16)
    with pytest.raises(ValueError):
        CS.consistency_score(v[:1], R[:1], t[:1], K[:1])
    with pytest.raises(ValueError):
        CS.consistency_score(v, R, t, K, every=8)           # nothing held out
    with pytest.raises(ValueError):
        CS.consistency_score(v, R, t, K, every=1)
    with pytest.raises(ValueError):
        CS.fit_field(v[..., :2], R, t, K)
    with pytest.raises(ValueError):
        CS.fit_field(v, R[:2], t[:2], K[:2])


# ---- 7. examples/consistency_srn.py on eval_srn.py's views ------------------------------------------------------------------
def test_consistency_script_end_to_end(tmp_path):
    pytest.importorskip('cv2')
    from tests.test_srn_data import _make_tree
    root, ck_dir, ev = str(tmp_path / 'cars'), str(tmp_path / 'ck'), str(tmp_path / 'eval')
    _make_tree(root, n_inst=2, n_views=8, H=64, W=64)
    params = P.XUNet().init({'params': 3}, {'x': np.zeros((1, 64, 64, 3), np.float32)}, zero_init=False)['params']
    P.checkpoint.save_checkpoint(ck_dir, params, step=0, prefix='model', add_device_axis=True)
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(repo, 'examples', 'eval_srn.py'), root, '--ckpt', ck_dir, '--side', '64',
                        '--steps', '4', '--source-view', '1', '--targets', '0', '--views-in-flight', '8', '--out', ev,
                        '--save-views'], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr

    def run(out, *extra):
        return subprocess.run([sys.executable, os.path.join(repo, 'examples', 'consistency_srn.py'), root, '--views',
                               os.path.join(ev, 'views'), '--side', '64', '--source-view', '1', '--every', '3', '--grid', '32',
                               '--iters', '100', '--rays', '2048', '--seed', '2', '--out', out, *extra],
                              capture_output=True, text=True, timeout=600)

    outs = [str(tmp_path / f'c{k}') for k in range(2)]
    for o in outs:
        r = run(o)
        assert r.returncode == 0, r.stdout + r.stderr
    lines = [json.loads(s) for s in open(os.path.join(outs[0], 'consistency.jsonl'))]
    assert [d['instance'] for d in lines] == ['obj0', 'obj1']
    for d in lines:
        assert d['views'] == [0, 2, 3, 4, 5, 6, 7] and d['held_out'] == [3, 6]
        vals = d['psnr'] + d['ssim'] + d['gt_psnr'] + d['gt_ssim'] + [d['mean_psnr'], d['gt_mean_psnr'], d['fit_loss'], d['gt_fit_loss']]
        assert all(math.isfinite(x) for x in vals), d
    summary = json.load(open(os.path.join(outs[0], 'summary.json')))
    assert json.loads(r.stdout.strip().splitlines()[-1])['n_instances'] == summary['n_instances'] == 2
    assert summary['n_held_out'] == 4 and all(math.isfinite(summary[k]) for k in ('mean_psnr', 'mean_ssim', 'gt_mean_psnr', 'gt_mean_ssim'))
    assert open(os.path.join(outs[0], 'consistency.jsonl'), 'rb').read() == open(os.path.join(outs[1], 'consistency.jsonl'), 'rb').read()

    r = run(str(tmp_path / 'bad'), '--every', '8')
    assert r.returncode != 0 and 'obj0' in r.stderr, r.stderr
