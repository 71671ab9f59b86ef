"""CPU checks of the camera-gradient math (xunet_backward_vjp_inputs): the oracle's ray generation is differentiable w.r.t. R, t
and K and matches finite differences, and the numpy restatements of the posenc Jacobian transpose and of the reduction from the
ray gradient to dR / dt / dK (what the CUDA epilogue and camera_grad_kernel compute) equal torch autograd."""
import numpy as np
import pytest
import torch

from oracle import xunet_ref as R
from tests import camera_grad_ref as CG

S, B = 16, 2


def _cams(seed=3):
    batch, _ = R.synthetic_batch(B, S, seed=seed)
    return {k: batch[k].clone() for k in CG.CAMERA_KEYS}


def _rays_value(cams, g_pos, g_dir, conv):
    r1 = R.camera_rays(cams['R1'], cams['t1'], cams['K'], S, S, conv)
    r2 = R.camera_rays(cams['R2'], cams['t2'], cams['K'], S, S, conv)
    return sum(((p * gp).sum() + (d * gd).sum()) for (p, d), gp, gd in zip((r1, r2), g_pos, g_dir))


@pytest.mark.parametrize('conv', ['v3d130_ij', 'opencv_uv'])
def test_camera_rays_autograd_matches_finite_differences(conv):
    cams = _cams()
    rng = np.random.RandomState(5)
    g_pos = [torch.from_numpy(rng.randn(B, S, S, 3)) for _ in range(2)]
    g_dir = [torch.from_numpy(rng.randn(B, S, S, 3)) for _ in range(2)]
    leaves = {k: v.clone().requires_grad_(True) for k, v in cams.items()}
    grads = dict(zip(leaves, torch.autograd.grad(_rays_value(leaves, g_pos, g_dir, conv), list(leaves.values()))))
    h = 1e-7
    for k in CG.CAMERA_KEYS:
        v = torch.from_numpy(rng.randn(*cams[k].shape))
        f = lambda sgn: float(_rays_value(dict(cams, **{k: cams[k] + sgn * h * v}), g_pos, g_dir, conv))
        fd = (f(1) - f(-1)) / (2 * h)
        an = float((grads[k] * v).sum())
        assert abs(fd - an) <= 1e-5 * max(abs(an), 1.0), (k, fd, an)


@pytest.mark.parametrize('conv', ['v3d130_ij', 'opencv_uv'])
def test_camera_reduction_equals_autograd(conv):
    cams = _cams(seed=4)
    rng = np.random.RandomState(6)
    d_rays = rng.randn(B, 2, S, S, 6)
    leaves = {k: v.clone().requires_grad_(True) for k, v in cams.items()}
    gp = [torch.from_numpy(d_rays[:, f, ..., :3]) for f in range(2)]
    gd = [torch.from_numpy(d_rays[:, f, ..., 3:]) for f in range(2)]
    grads = dict(zip(leaves, torch.autograd.grad(_rays_value(leaves, gp, gd, conv), list(leaves.values()))))
    mine = CG.camera_reduce(d_rays, (cams['R1'].numpy(), cams['R2'].numpy()), cams['K'].numpy(), S, conv)
    for k in CG.CAMERA_KEYS:
        ref = grads[k].numpy()
        assert np.abs(mine[k] - ref).max() <= 1e-10 * max(np.abs(ref).max(), 1.0), k


def _posenc_fixed_args(x, nd):
    """posenc_nerf(x, 0, nd) in fp64 with the fp32 arguments held: arg = 2^k x + (fl32 argument - 2^k x) with the bracket a
    constant, so autograd differentiates exactly the linearisation at the forward's arguments."""
    x32 = x.detach().to(torch.float32)
    sc32 = torch.tensor([2.0 ** i for i in range(nd)], dtype=torch.float32)
    xb32 = (x32[..., None, :] * sc32[:, None]).reshape(*x.shape[:-1], -1)
    a32 = torch.cat([xb32, xb32 + torch.tensor(np.pi / 2, dtype=torch.float32)], -1).double()
    sc = sc32.double()
    xb = (x[..., None, :] * sc[:, None]).reshape(*x.shape[:-1], -1)
    lin = torch.cat([xb, xb], -1)
    return torch.cat([x, torch.sin(lin + (a32 - lin.detach()))], -1)


@pytest.mark.parametrize('nd', [15, 8])
def test_posenc_jacobian_transpose_equals_autograd(nd):
    rng = np.random.RandomState(nd)
    v = torch.from_numpy(rng.uniform(-1.5, 1.5, (64, 3)).astype(np.float32)).double()
    g = torch.from_numpy(rng.randn(64, 3 + 6 * nd))
    x = v.clone().requires_grad_(True)
    want, = torch.autograd.grad((_posenc_fixed_args(x, nd) * g).sum(), [x])
    got = CG.posenc_jt(g.numpy(), v.numpy(), nd)
    assert np.abs(got - want.numpy()).max() <= 1e-10 * np.abs(want.numpy()).max()
    # the oracle's own posenc_nerf: same values; its backward runs through fp32 casts, so it agrees to fp32 rounding only
    x = v.clone().requires_grad_(True)
    assert torch.equal(_posenc_fixed_args(x, nd).detach(), R.posenc_nerf(v, 0, nd))
    oracle, = torch.autograd.grad((R.posenc_nerf(x, 0, nd) * g).sum(), [x])
    assert np.abs(got - oracle.numpy()).max() <= 1e-5 * np.abs(got).max()
