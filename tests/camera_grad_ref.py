"""References of the camera gradient (xunet_backward_vjp_inputs): the posenc Jacobian transpose and the reduction of the ray
gradient to dR / dt / dK restated in numpy fp64, and torch autograd through the oracle with the cameras (or the rays) as leaves."""
from collections import OrderedDict

import numpy as np
import torch

from oracle import xunet_ref as R

CAMERA_KEYS = ('R1', 't1', 'R2', 't2', 'K')


def posenc_jt(g, v, nd):
    """J^T g of posenc_nerf(v, 0, nd) at fixed fp32 arguments: g (..., 3 + 6 nd) fp64, v (..., 3) the fp32 ray components.
    Entry of channel sin(2^k v_d): 2^k cos(fl32(2^k v_d)); of the shifted channel: 2^k cos(fl32(fl32(2^k v_d) + pi/2))."""
    v32 = np.asarray(v, np.float32)
    g = np.asarray(g, np.float64)
    out = g[..., :3].copy()
    for k in range(nd):
        xb = v32 * np.float32(2.0 ** k)
        sh = xb + np.float32(np.pi / 2)
        out += 2.0 ** k * np.cos(xb.astype(np.float64)) * g[..., 3 + 3 * k: 6 + 3 * k]
        out += 2.0 ** k * np.cos(sh.astype(np.float64)) * g[..., 3 + 3 * nd + 3 * k: 6 + 3 * nd + 3 * k]
    return out


def rays_jt(g144, pos, dirs):
    """(…, 144) posenc gradient -> (…, 6) [d pos | d dir]."""
    return np.concatenate([posenc_jt(g144[..., :93], pos, 15), posenc_jt(g144[..., 93:], dirs, 8)], axis=-1)


def camera_reduce(d_rays, Rs, K, S, convention='v3d130_ij'):
    """d_rays (B,2,S,S,6) -> {'R1','t1','R2','t2','K'} in fp64: dt = sum d pos; with c = K^-1 p, w = R c, dir = w/|w|:
    d_w = (d dir - dir (dir . d dir)) / |w|, dR = sum d_w c^T, dK^-1 = sum (R^T d_w) p^T over both cameras,
    dK = -K^-T dK^-1 K^-T."""
    d_rays = np.asarray(d_rays, np.float64)
    K = np.asarray(K, np.float64)
    ii, jj = np.meshgrid(np.arange(S) + 0.5, np.arange(S) + 0.5, indexing='ij')
    p0, p1 = (ii, jj) if convention == 'v3d130_ij' else (jj, ii)
    p = np.stack([p0, p1, np.ones_like(p0)], -1)                        # (S,S,3)
    Kinv = np.linalg.inv(K)                                               # (B,3,3)
    c = np.einsum('bij,hwj->bhwi', Kinv, p)
    out, gkinv = {}, 0.0
    for f, (rk, tk) in enumerate((('R1', 't1'), ('R2', 't2'))):
        Rm = np.asarray(Rs[f], np.float64)
        w = np.einsum('bij,bhwj->bhwi', Rm, c)
        nw = np.linalg.norm(w, axis=-1, keepdims=True)
        d = w / nw
        dd = d_rays[:, f, ..., 3:]
        dw = (dd - d * (d * dd).sum(-1, keepdims=True)) / nw
        out[tk] = d_rays[:, f, ..., :3].sum((1, 2))
        out[rk] = np.einsum('bhwi,bhwj->bij', dw, c)
        gkinv = gkinv + np.einsum('bhwi,hwj->bij', np.einsum('bji,bhwj->bhwi', Rm, dw), p)
    out['K'] = -np.einsum('bji,bjk,blk->bil', Kinv, gkinv, Kinv)
    return out


def d_rays_ref(eng, flat, comps, cond, bf16):
    """fp64 ray gradient from the engine's own inputs: each level's output gradient as the engine stored it
    (read_tap('pose_emb_l', grad=True)), its kernel (rounded to bf16 in bf16 mode), a strided conv-transpose with XLA SAME
    padding, then J^T at the fp32 ray components comps = (pos, dir), each (B,2,S,S,3)."""
    S, B = eng.S, eng.B
    g = torch.zeros(2 * B, 144, S, S, dtype=torch.float64)
    for l in range(len(eng.cfg.ch_mult)):
        dy = eng.read_tap(f'pose_emb_{l}', grad=True).double().cpu().permute(0, 3, 1, 2)
        shape, off = eng.spec[f'ConditioningProcessor_0/Conv_{l}/kernel']
        w = flat[off:off + int(np.prod(shape))].view(shape)[0]
        if bf16:
            w = w.to(torch.bfloat16)
        w = w.double().cpu().permute(3, 2, 0, 1)                           # (E, 144, 3, 3)
        s = 2 ** l
        lo, hi = R.same_pad(S, 3, s)
        gp = torch.nn.grad.conv2d_input((2 * B, 144, S + lo + hi, S + lo + hi), w, dy, stride=s)
        g += gp[:, :, lo:lo + S, lo:lo + S]
    g = g.permute(0, 2, 3, 1).reshape(B, 2, S, S, 144).numpy()
    out = rays_jt(g, comps[0], comps[1])
    out[np.asarray(cond) == 0] = 0.0
    return out


class PoseSTE(R.Bf16Emulation):
    """Bf16Emulation whose bf16 store of the posenc tensor (B,2,S,S,144) is straight-through (_RoundSTE): the value is rounded,
    the gradient reaches the rays unrounded, as the engine's fp32 J^T epilogue does."""

    def store(self, t):
        if t.dim() == 5 and t.shape[-1] == R.POSE_EMB_DIM:
            return R._RoundSTE.apply(t)
        return R._Store.apply(t)


def camera_vjp(params, batch, cond_mask, d_eps, cfg, *, rays=None, emu=None, convention='v3d130_ij'):
    """Autograd of L = <d_eps, eps_hat> through the oracle with the cameras (or, given rays ((pos1, dir1), (pos2, dir2)), the
    rays) as leaves: returns an OrderedDict of their gradients ('R1'...'K', or 'rays' (B,2,S,S,6))."""
    p = R.nest(OrderedDict((k, v.detach()) for k, v in R.flatten(params).items()))
    if rays is None:
        leaves = OrderedDict((k, batch[k].detach().clone().requires_grad_(True)) for k in CAMERA_KEYS)
        eps = R.xunet_forward(p, dict(batch, **leaves), cond_mask, cfg, emu=emu, ray_convention=convention)
        grads = torch.autograd.grad((eps * d_eps.to(eps.dtype)).sum(), list(leaves.values()))
        return OrderedDict(zip(leaves, grads))
    leaf = torch.stack([torch.cat([pp, dd], -1) for pp, dd in rays], 1).detach().clone().requires_grad_(True)
    rr = tuple((leaf[:, f, ..., :3], leaf[:, f, ..., 3:]) for f in range(2))
    eps = R.xunet_forward(p, batch, cond_mask, cfg, emu=emu, rays=rr)
    g, = torch.autograd.grad((eps * d_eps.to(eps.dtype)).sum(), [leaf])
    return OrderedDict(rays=g)
