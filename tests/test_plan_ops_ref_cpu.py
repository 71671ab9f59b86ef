"""CPU checks of tests/plan_ops_ref.py, the fp64 references and per-element bounds of the conditioning, resampling, concat and
loss launches: the references against the oracle and torch autograd, the bounds accepting a result that carries nothing but
its final rounding, and rejecting each of a set of subtle kernel or plan bugs."""
import math

import numpy as np
import pytest
import torch

from oracle import xunet_ref as R
from tests import launch_ref as L
from tests import plan_ops_ref as O

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _f32(t):
    return t.to(torch.float32).to(F64)


def _bf(t):
    return t.to(torch.bfloat16).to(F64)


def _cams(B, g, skew=0.3):
    """fp32-valued rotations, centres up to |t| = 8 and intrinsics with cx != cy and a non-zero skew"""
    q, _ = torch.linalg.qr(torch.randn(B, 3, 3, generator=g, dtype=F64))
    t = _f32(torch.randn(B, 3, generator=g, dtype=F64) * 3.).clamp(-8., 8.)
    K = torch.tensor([[70., skew, 30.], [0., 65., 34.], [0., 0., 1.]], dtype=F64).repeat(B, 1, 1)
    K[:, 0, 0] += torch.rand(B, generator=g, dtype=F64)
    return _f32(q), t, _f32(K)


# ---- the references against the oracle and autograd ----
@pytest.mark.parametrize('E', [32, 1024])
def test_posenc_ddpm_matches_oracle(E):
    l = torch.tensor([-25., -20., -3.5, 0., 4.25, 19.9, 30.], dtype=F64)
    ref, _ = O.posenc_ddpm_check(l, E)
    t = 2. * torch.atan(torch.exp(-l.clamp(-20., 20.) / 2.)) / math.pi
    assert torch.allclose(ref, R.posenc_ddpm(t, E, max_time=1.), rtol=0, atol=1e-12)


@pytest.mark.parametrize('convention', [0, 1])
def test_rays_and_posenc_match_oracle(convention):
    g = _g(2)
    Rm, t, K = _cams(3, g)
    S = 6
    kinv, _ = O.kinv_check(K.reshape(-1, 9))
    d, _ = O.ray_dirs(kinv, Rm, S, convention)
    _, dref = R.camera_rays(Rm, t, K, S, S, ['v3d130_ij', 'opencv_uv'][convention])
    assert torch.allclose(d, dref, rtol=0, atol=1e-12)
    v = _f32(torch.randn(4, 5, 3, generator=g, dtype=F64) * 4.)
    for nd in (8, 15):
        assert torch.allclose(O.posenc_nerf32(v, nd), R.posenc_nerf(v, 0, nd), rtol=0, atol=1e-12)
        ex, _ = O.posenc_nerf_exact(v, torch.zeros_like(v[..., :1]), nd)
        # exact sin / cos of 2^k v: differs from the fp32-argument restatement by the rounding of the add of pi/2 alone
        assert torch.allclose(ex[..., :3 + 3 * nd], O.posenc_nerf32(v, nd)[..., :3 + 3 * nd], rtol=0, atol=1e-12)


def test_pose_embedding_matches_oracle_conditioning():
    g = _g(3)
    B, S = 3, 5
    R1, t1, K = _cams(B, g)
    R2, t2, _ = _cams(B, g)
    cond = torch.tensor([1., 0., 1.], dtype=F64)
    pe = torch.randn(S, S, 144, generator=g, dtype=F64)
    rf, ro = torch.randn(144, generator=g, dtype=F64), torch.randn(144, generator=g, dtype=F64)
    kinv = torch.linalg.inv(K).reshape(B, 9)
    ref, bound = O.pose_emb_check(0, R1, t1, R2, t2, kinv, cond, S, 0, pe, rf, ro)
    # the oracle's conditioning() up to the level convs, from its own pieces
    embs = []
    for Rk, tk in ((R1, t1), (R2, t2)):
        pos, d = R.camera_rays(Rk, tk, K, S, S)
        embs.append(torch.cat([R.posenc_nerf(pos, 0, 15), R.posenc_nerf(d, 0, 8)], -1))
    pose = torch.stack(embs, 1)
    pose = torch.where(cond.reshape(B, 1, 1, 1, 1).bool(), pose, torch.zeros_like(pose)) + pe[None, None]
    pose = pose + torch.stack([rf, ro])[None, :, None, None, :]
    # the oracle rounds its fp64 directions to fp32 before the sin arguments, as the kernel does: within the bound
    assert _in(pose.reshape(2 * B, S, S, 144), ref, bound)


def test_logsnr_backward_matches_autograd():
    g = _g(4)
    B, E = 3, 16
    pe = torch.randn(B, E, generator=g, dtype=F64)
    w0, w1 = (torch.randn(E, E, generator=g, dtype=F64, requires_grad=True) for _ in range(2))
    b0, b1 = (torch.randn(E, generator=g, dtype=F64, requires_grad=True) for _ in range(2))
    h1 = (pe @ w0 + b0).detach().requires_grad_(True)
    lemb = O.swish(h1) @ w1 + b1
    dl = torch.randn(B, E, generator=g, dtype=F64)
    gh1, gw1, gb1 = torch.autograd.grad(lemb, [h1, w1, b1], dl)
    h0 = h1.detach()
    chk = dict((n, r) for n, r, _ in O.logsnr_bwd_check(dl, w1.detach(), pe, h0, gh1))
    assert torch.allclose(chk['dh1'], gh1) and torch.allclose(chk['dw1'], gw1) and torch.allclose(chk['db1'], gb1)
    gw0, gb0 = torch.autograd.grad(pe @ w0 + b0, [w0, b0], gh1)
    assert torch.allclose(chk['dw0'], gw0) and torch.allclose(chk['db0'], gb0)


def test_film_emb_resample_and_loss_backward_match_autograd():
    g = _g(5)
    N, HW, E = 4, 6, 8
    lemb = torch.randn(N // 2, E, generator=g, dtype=F64, requires_grad=True)
    pe = torch.randn(N, HW, E, generator=g, dtype=F64, requires_grad=True)
    y, _ = O.film_emb_check(lemb, pe, False)
    ds = torch.randn(N, HW, E, generator=g, dtype=F64)
    gl, gp = torch.autograd.grad(y, [lemb, pe], ds)
    dz, _, dl, _ = O.film_emb_bwd_check(lemb.detach(), pe.detach(), ds, False, torch.zeros(N // 2, E, dtype=F64))
    assert torch.allclose(dz, gp) and torch.allclose(dl, gl)
    # resample: the forward against the oracle; the backward the engine runs (pool <-> 0.25 replicate, replicate <-> 2x2 sum)
    x = torch.randn(2, 4, 6, 8, generator=g, dtype=F64, requires_grad=True)
    down, _ = O.resample_check(x, 1, 0.25, False)
    assert torch.allclose(down, R.avgpool_downsample(x.reshape(1, 2, 4, 6, 8)).reshape(2, 2, 3, 8))
    up, _ = O.resample_check(x, 0, 1., False)
    assert torch.allclose(up, R.nearest_neighbor_upsample(x.reshape(1, 2, 4, 6, 8)).reshape(2, 8, 12, 8))
    for fwd, adj, shape in ((lambda t: O.resample_check(t, 1, 0.25, False)[0], lambda d: O.resample_check(d, 0, 0.25, False)[0],
                             (2, 2, 3, 8)),
                            (lambda t: O.resample_check(t, 0, 1., False)[0], lambda d: O.resample_check(d, 1, 1., False)[0],
                             (2, 8, 12, 8))):
        dy = torch.randn(*shape, generator=g, dtype=F64)
        gx, = torch.autograd.grad(fwd(x), [x], dy)
        assert torch.allclose(adj(dy), gx)
    # loss = ||eps - noise||
    eps = torch.randn(2, 3, 3, 3, generator=g, dtype=F64, requires_grad=True)
    noise = torch.randn(2, 3, 3, 3, generator=g, dtype=F64)
    ge, = torch.autograd.grad(R.loss_fn(eps, noise), [eps])
    _, _, loss, _, dO, _ = O.loss_check(eps.detach(), noise, False)
    assert torch.allclose(loss, R.loss_fn(eps.detach(), noise)) and torch.allclose(dO[1::2], ge) and not dO[0::2].any()


# ---- the bounds accept a result carrying only its final rounding, and reject each bug ----
def _in(got, ref, bound):
    return L.within(got, ref, bound)


def _logsnr_case(B, E, seed=6):
    g = _g(seed)
    l = _f32(torch.cat([torch.tensor([-24., 23.]), torch.randn(B - 2, generator=g, dtype=F64) * 8.]))
    w0 = _f32(torch.randn(E, E, generator=g, dtype=F64) / math.sqrt(E))
    w1 = _f32(torch.randn(E, E, generator=g, dtype=F64) / math.sqrt(E))
    b0, b1 = _f32(torch.randn(E, generator=g, dtype=F64) * .3), _f32(torch.randn(E, generator=g, dtype=F64) * .3)
    pe = _f32(O.posenc_ddpm_check(l, E)[0])
    h1 = _f32(pe @ w0 + b0)
    return l, w0, b0, w1, b1, pe, h1


@pytest.mark.parametrize('E', [32, 1024])
def test_logsnr_bounds(E):
    l, w0, b0, w1, b1, pe, h1 = _logsnr_case(8, E)
    chk = O.logsnr_fwd_check(l, w0, b0, w1, b1, pe, h1)
    for name, ref, bound in chk:
        assert _in(_f32(ref), ref, bound), name
    # the first 32-column block of Dense_0 computed with the next block's weights (E = 32: shifted by one column)
    name, ref, bound = chk[1]
    bad = ref.clone()
    cols = (torch.arange(32) + (32 if E > 32 else 1)) % E
    bad[:, :32] = _f32(pe @ w0[:, cols] + b0[cols])
    assert not _in(bad, ref, bound)
    # backward: the last sample dropped from the bias sums
    g = _g(7)
    dl = _f32(torch.randn(8, E, generator=g, dtype=F64) + 0.2)
    dh1 = _f32(O.swish_grad(h1) * (dl @ w1.T))
    bwd = O.logsnr_bwd_check(dl, w1, pe, h1, dh1)
    for name, ref, bound in bwd:
        assert _in(_f32(ref), ref, bound), name
    d = {n: (r, b) for n, r, b in bwd}
    assert not _in(dl[:-1].sum(0), *d['db1'])
    assert not _in(dh1[:-1].sum(0), *d['db0'])


def test_logsnr_bound_rejects_the_frequency_of_half_instead_of_half_minus_one():
    E = 1024
    l = _f32(torch.linspace(-20., 20., 9, dtype=F64))
    ref, bound = O.posenc_ddpm_check(l, E)
    half = E // 2
    t = O.logsnr_time(l)[:, None]
    f = torch.exp(-torch.arange(half, dtype=F64) * (math.log(10000.) / half))
    bad = torch.cat([torch.sin(t * f), torch.cos(t * f)], -1)
    assert not _in(bad, ref, bound)


def test_kinv_bound_rejects_a_transposed_inverse():
    g = _g(8)
    _, _, K = _cams(4, g)
    ref, bound = O.kinv_check(K.reshape(-1, 9))
    assert _in(_f32(ref), ref, bound)
    bad = ref.reshape(-1, 3, 3).transpose(1, 2).reshape(-1, 9)
    assert not _in(bad, ref, bound)


@pytest.mark.parametrize('dtype', [0, 1])
def test_pose_emb_bounds(dtype):
    g = _g(9)
    B, S = 2, 20
    R1, t1, K = _cams(B, g)
    R2, t2, _ = _cams(B, g)
    t1[0] = torch.tensor([8., -7.9, 7.5], dtype=F64)
    cond = torch.tensor([1., 1.], dtype=F64)
    kinv = _f32(torch.linalg.inv(K).reshape(B, 9))
    ref, bound = O.pose_emb_check(dtype, R1, t1, R2, t2, kinv, cond, S, 0)
    st = (lambda t: _bf(t)) if dtype == 1 else _f32
    assert _in(st(ref), ref, bound)
    # a transposed K^-1 moves the directions
    bad, _ = O.pose_emb_check(dtype, R1, t1, R2, t2, kinv.reshape(B, 3, 3).transpose(1, 2).reshape(B, 9), cond, S, 0)
    assert not _in(st(bad), ref, bound)
    if dtype == 0:
        # the fp32 verify plan: the sin channels at the kernel's own fp32 directions, and cos(2^k v) in place of
        # sin(fl32(2^k v + pi/2)) in every shifted channel (origin and direction)
        dirs = torch.stack([_f32(O.ray_dirs(kinv, Rk, S, 0)[0]) for Rk in (R1, R2)], 1)
        ref2, bound2 = O.pose_emb_check(0, R1, t1, R2, t2, kinv, cond, S, 0, dirs32=dirs)
        assert _in(_f32(ref2), ref2, bound2)
        bad = ref2.clone().reshape(B, 2, S, S, 144)
        for f, tk in enumerate((t1, t2)):
            v = torch.cat([tk[:, None, None, :].expand(B, S, S, 3), dirs[:, f]], -1)
            for nd, c0, vv in ((15, 0, v[..., :3]), (8, 93, v[..., 3:])):
                xb = torch.cat([vv * 2. ** k for k in range(nd)], -1)
                bad[:, f, ..., c0 + 3 + 3 * nd:c0 + 3 + 6 * nd] = torch.cos(xb)
        assert not _in(bad.reshape(ref2.shape), ref2, bound2)


def test_film_emb_bounds_reject_a_missing_pixel_block_of_dlemb():
    g = _g(10)
    N, HW, E = 4, 400, 32
    lemb = _f32(torch.randn(N // 2, E, generator=g, dtype=F64))
    pe = _bf(torch.randn(N, HW, E, generator=g, dtype=F64) + 0.3)
    ds = _bf(torch.randn(N, HW, E, generator=g, dtype=F64) + 0.2)
    prior = _f32(torch.randn(N // 2, E, generator=g, dtype=F64))
    ref, bound = O.film_emb_check(lemb, pe, True)
    assert _in(_bf(ref), ref, bound)
    dz, bdz, dl, bdl = O.film_emb_bwd_check(lemb, pe, ds, True, prior)
    assert _in(_bf(dz), dz, bdz) and _in(_f32(dl), dl, bdl)
    # 256 pixels of sample 1 (one block of emb_bwd_kernel at this shape), or only its last pixel, never summed
    P = 2 * HW
    for lo, hi in ((256, 512), (P - 1, P)):
        bad = dl.clone()
        bad[1] -= dz.reshape(N // 2, P, E)[1, lo:hi].sum(0)
        assert not _in(bad, dl, bdl)


def test_copy_bound_rejects_an_accumulate_read_without_dst_off():
    g = _g(11)
    npix, Cs, Cd, so, do, Cc = 10, 96, 32, 64, 0, 32
    src = torch.randn(npix, Cs, generator=g).to(torch.bfloat16)
    dst = torch.randn(npix, Cd, generator=g).to(torch.bfloat16)
    # the backward copy into the second input (dst_off 0) and the forward copy of b into y (dst_off > 0)
    for Cs_, Cd_, so_, do_ in ((Cs, Cd, so, do), (32, 96, 0, 64)):
        s = src[:, :Cs_]
        d = torch.randn(npix, Cd_, generator=g).to(torch.bfloat16)
        ex = O.copy_channels_exact(s, d, Cs_, Cd_, so_, do_, Cc, 1)
        bad = d.clone()
        bad[:, do_:do_ + Cc] = (s[:, so_:so_ + Cc].float() + d[:, 0:Cc].float()).to(torch.bfloat16)
        assert torch.equal(ex[:, do_:do_ + Cc], (s[:, so_:so_ + Cc].float() + d[:, do_:do_ + Cc].float()).to(torch.bfloat16))
        assert torch.equal(bad, ex) == (do_ == 0)
    del dst


def test_resample_bound_rejects_an_adjoint_without_its_alias_scale():
    g = _g(12)
    dy = _bf(torch.randn(4, 8, 8, 32, generator=g, dtype=F64) + 0.1)
    prior = _bf(torch.randn(4, 16, 16, 32, generator=g, dtype=F64))
    gs = float(np.float32(1 / math.sqrt(2)))
    scale = float(np.float32(np.float32(0.25) * np.float32(gs)))
    ref, bound = O.resample_check(dy, 0, scale, True, prior)
    assert _in(_bf(ref), ref, bound)
    bad, _ = O.resample_check(dy, 0, 0.25, True, prior)
    assert not _in(_bf(bad), ref, bound)
    r2, b2 = O.scale_add_check(dy, gs, True, _bf(torch.randn(4, 8, 8, 32, generator=g, dtype=F64)))
    assert _in(_bf(r2), r2, b2)


def test_loss_bound_rejects_a_nan_from_a_zero_loss():
    g = _g(13)
    eps = _f32(torch.randn(2, 8, 8, 3, generator=g, dtype=F64))
    noise = _f32(torch.randn(2, 8, 8, 3, generator=g, dtype=F64))
    ss, bss, loss, bl, dO, bdO = O.loss_check(eps, noise, True)
    assert _in(_f32(ss), ss, bss) and _in(_f32(loss), loss, bl) and _in(_bf(dO), dO, bdO)
    ss, bss, loss, bl, dO, bdO = O.loss_check(eps, eps, True)
    assert float(loss) == 0. and _in(torch.zeros_like(dO), dO, bdO)
    nan = torch.zeros_like(dO)
    nan[1::2] = float('nan')     # (eps - noise) / loss without the loss > 0 guard: 0 / 0
    assert not _in(nan, dO, bdO)
