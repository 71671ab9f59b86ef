"""The GroupNorm path kernel by kernel against fp64 (tests/groupnorm_ref.py), through the operator entry points that run the
engine's launches: the producers' statistics (conv EPI 1, attention, the statistics kernel), the apply kernels, the fused
backward epilogues of the consumer conv's data gradient (EPI 2, EPI 3) and the backward apply kernels.

Every stage is checked on the kernel's own inputs (what the previous stage stored) with bounds tight enough that one wrong
column, channel, group, sample or frame fails:
  * sums (cstats, bcs, stats, bstats): |got - ref| <= rel * sum|terms|, ref the fp64 sum over the stored tensors;
  * tensors, per element: |got - ref| <= 2^-8 |ref| + floor (bf16 store: one rounding, 2^-9 relative, with margin; fp32:
    1e-5 |ref|), the floor the fp32 arithmetic's error relative to the magnitude of the terms that cancel, derived where it
    is used.
A chain check then runs the fp64 reference from the bf16-rounded inputs alone (rel-L2).
The fp64 references run on the GPU in float64 (test-side arithmetic only)."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import groupnorm_ref as G
from tests import launch_ref as L
from tests.util import keep_mask

pytestmark = pytest.mark.gpu

DT = {0: torch.float32, 1: torch.bfloat16}
F64 = torch.float64
BF_REL = 2. ** -8        # a bf16 store: one rounding, 2^-8 relative (8 significand bits); the fp32 work before it is in the floors
F32_REL = 1e-5
SEED = 0x5DEECE66D


def _s():
    return torch.cuda.current_stream().cuda_stream


def _rand(shape, g, scale=1., shift=0.):
    return (torch.randn(shape, generator=g, dtype=F64) * scale + shift).cuda()


def _q(t, dtype):
    """round to the storage type and back to fp64: the kernel's input"""
    return t.to(DT[dtype]).to(F64)


def _dev(t, dtype):
    """the device copy in the storage type (None stays None).  Bind it to a name before passing data_ptr() to a call: a
    temporary would return its memory to the allocator before the asynchronous launch reads it."""
    return None if t is None else t.to(DT[dtype]).contiguous()


def _p(t):
    return None if t is None else t.data_ptr()


def rel_l2(a, b):
    a, b = a.to(F64), b.to(F64)
    return float(torch.linalg.norm(a - b) / torch.linalg.norm(b))


def _seed_dev(seed=SEED):
    return torch.tensor([seed], dtype=torch.int64, device='cuda')


def assert_elems(got, ref, floor, rel, what):
    """|got - ref| <= rel |ref| + floor, element by element; the message names the worst element"""
    got = got.to(F64)
    err = (got - ref).abs()
    bound = rel * ref.abs() + floor
    bad = err > bound
    if bool(bad.any()):
        i = int(torch.argmax((err - bound).reshape(-1)))
        idx = np.unravel_index(i, tuple(ref.shape))
        raise AssertionError(f'{what}: {int(bad.sum())} of {ref.numel()} elements out of bounds; worst at {idx}: got '
                             f'{float(got.reshape(-1)[i]):.6g}, ref {float(ref.reshape(-1)[i]):.6g}, bound '
                             f'{float(bound.reshape(-1)[i]):.3g}')


def assert_sums(got, ref, terms, rel, what):
    """|got - ref| <= rel * sum|terms| + 1e-30 per sum"""
    assert_elems(got, ref, rel * terms + 1e-30, 0., what)


def _conv_ref(x, w, ks, nseg=1):
    """Flax SAME conv (stride 1) in fp64: x (N,H,W,Ci), w (taps, Ci, Co) fp64 -> (N,H,W,Co) (no bias); nseg: the Co segments of
    a 1x1 are the weight leaves [seg][Ci][segw] laid end to end."""
    N, H, W, Ci = x.shape
    if ks == 1:
        if nseg == 1:
            return x @ w[0]
        segw = w.numel() // (Ci * nseg)
        ws = w.reshape(nseg, Ci, segw)
        return torch.cat([x @ ws[s] for s in range(nseg)], dim=-1)
    Co = w.shape[-1]
    wt = w.reshape(3, 3, Ci, Co).permute(3, 2, 0, 1)
    return F.conv2d(x.permute(0, 3, 1, 2), wt, padding=1).permute(0, 2, 3, 1)


def _dgrad_ref(dy, w, ks, C, nseg=1):
    """data gradient of _conv_ref: dy (N,H,W,Co) -> (N,H,W,C)"""
    N, H, W, Co = dy.shape
    if ks == 1:
        ws = w.reshape(nseg, C, Co // nseg)
        return sum(dy[..., s * (Co // nseg):(s + 1) * (Co // nseg)] @ ws[s].T for s in range(nseg))
    wt = w.reshape(3, 3, C, Co).permute(3, 2, 0, 1)
    return torch.nn.grad.conv2d_input((N, C, H, W), wt, dy.permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)


# conv accumulation floor of a K-term fp32 sum: L.acc_floor(K) of sum|terms| (tests/launch_ref.py derives it), 2^-16 at
# K = 9 * 256 and less for the shorter reductions, still ~10^-3 of a typical output, so a misplaced element cannot hide in it.
CONV_FLOOR = L.acc_floor


# ======================================================================================================================
# producers: conv EPI 1 / statistics kernel, attention statistics
# ======================================================================================================================
CONV_STATS_CASES = [
    # dtype, impl, N, H, W, Ci, Co, ks, residual, alpha
    (1, 1, 6, 16, 16, 32, 64, 3, True, 1 / math.sqrt(2)),     # halo, BN 32, two n-tiles, residual
    (1, 1, 6, 8, 8, 96, 64, 3, False, 1.),                    # no halo (8x8 images, two per tile), BN 32
    (1, 1, 16, 4, 4, 64, 64, 3, True, 1 / math.sqrt(2)),      # 16-pixel images: TN = 8, B = 8 samples per tile
    (1, 1, 6, 8, 8, 64, 256, 1, False, 1.),                   # 1x1: TMA-store epilogue, eight n-tiles
    (1, 1, 4, 64, 64, 32, 128, 3, True, 1 / math.sqrt(2)),    # halo, BN 64, two CTAs per SM
    (1, 1, 6, 64, 64, 32, 128, 3, False, 1.),                 # halo, BN 128, one CTA per SM, persistent
    (0, 0, 6, 8, 8, 32, 64, 3, True, 1 / math.sqrt(2)),       # fp32 SIMT conv + statistics kernel
    (1, 0, 6, 8, 8, 32, 64, 3, True, 1 / math.sqrt(2)),       # bf16 SIMT conv + statistics kernel
    (1, 2, 6, 8, 8, 3, 32, 3, False, 1.),                     # 3-channel input conv + statistics kernel
]


def _run_conv_stats(lib, case):
    dtype, impl, N, H, W, Ci, Co, ks, has_res, alpha = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFFFF)
    taps = ks * ks
    x = _q(_rand((N, H, W, Ci), g), dtype)
    w = _rand((taps, Ci, Co), g, 1 / math.sqrt(taps * Ci)).float()
    b = _rand((Co,), g, 0.3).float()
    # a per-sample offset so that every sample's statistics differ (a routing error between samples shows)
    res = _q(_rand((N, H, W, Co), g) + torch.arange(N, device='cuda', dtype=F64).div(2, rounding_mode='floor')[:, None, None, None],
             dtype) if has_res else None
    y = torch.zeros(N, H, W, Co, dtype=DT[dtype], device='cuda')
    cs = torch.zeros(N // 2, Co, 2, dtype=torch.float32, device='cuda')
    xd, rd = _dev(x, dtype), _dev(res, dtype)
    rc = lib.xunet_op_conv_stats(dtype, impl, xd.data_ptr(), w.data_ptr(), b.data_ptr(), _p(rd), y.data_ptr(), cs.data_ptr(),
                                 N, H, W, Ci, Co,
                                 ks, alpha, _s())
    assert rc == 0, lib.xunet_last_error()
    return x, w, b, res, y, cs


@pytest.mark.parametrize('case', CONV_STATS_CASES)
def test_conv_stats(lib, case):
    dtype, impl, N, H, W, Ci, Co, ks, has_res, alpha = case
    x, w, b, res, y, cs = _run_conv_stats(lib, case)
    torch.cuda.synchronize()
    # stage: the statistics of what was STORED, in fp64.  The epilogue sums 16-column x 32-row slices in fp32 (a few tens of
    # terms, <= 2^-19 sum|terms|) and adds the slices in fp64: 1e-6 sum|terms|.
    y64 = y.to(F64)
    assert_sums(cs.to(F64), G.cstats(y64), G.cstats(y64.abs()), 1e-6, 'cstats')
    # chain: y against the fp64 conv of the bf16 inputs.  The tensor-core path multiplies the bf16 weight shadow, the SIMT paths
    # the fp32 weights.
    wr = (w.to(torch.bfloat16) if impl == 1 else w).to(F64)
    ref = _conv_ref(x, wr, ks) + b.to(F64)
    mag = _conv_ref(x.abs(), wr.abs(), ks) + b.to(F64).abs()
    if has_res:
        ref, mag = ref + res, mag + res.abs()
    ref, mag = ref * alpha, mag * alpha
    assert_elems(y, ref, CONV_FLOOR(ks * ks * Ci) * mag, BF_REL if dtype == 1 else F32_REL, 'y')
    assert rel_l2(y, ref) < (6e-3 if dtype == 1 else 1e-5)


ATTN_CASES = [
    # dtype, impl, N, L, C, heads, cross
    (1, 1, 4, 128, 64, 4, 0),      # head_dim 16
    (1, 1, 4, 128, 64, 2, 1),      # head_dim 32, cross
    (1, 1, 4, 256, 128, 2, 0),     # head_dim 64
    (1, 1, 6, 128, 256, 2, 1),     # head_dim 128, cross, B = 3
    (1, 0, 4, 64, 64, 2, 1),       # SIMT + statistics kernel
    (0, 0, 4, 64, 64, 2, 0),
]


def _attn_ref(qkv, res, heads, cross):
    N, L, C3 = qkv.shape
    C = C3 // 3
    hd = C // heads
    q, k, v = [t.reshape(N, L, heads, hd) for t in torch.split(qkv, C, dim=-1)]
    if cross:
        perm = torch.arange(N, device=qkv.device) ^ 1
        k, v = k[perm], v[perm]
    p = torch.softmax(torch.einsum('nqhd,nkhd->nhqk', q / math.sqrt(hd), k), dim=-1)
    return (torch.einsum('nhqk,nkhd->nqhd', p, v).reshape(N, L, C) + res) / math.sqrt(2)


@pytest.mark.parametrize('case', ATTN_CASES)
def test_attention_stats(lib, case):
    dtype, impl, N, L, C, heads, cross = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFFFF)
    qkv = _q(_rand((N, L, 3 * C), g, 1.5), dtype)
    res = _q(_rand((N, L, C), g) + torch.arange(N, device='cuda', dtype=F64)[:, None, None] * 0.5, dtype)
    out = torch.zeros(N, L, C, dtype=DT[dtype], device='cuda')
    lse = torch.zeros(N, heads, L, dtype=torch.float32, device='cuda')
    cs = torch.zeros(N // 2, C, 2, dtype=torch.float32, device='cuda')
    qd, rd = _dev(qkv, dtype), _dev(res, dtype)
    assert lib.xunet_op_attention_stats(dtype, impl, qd.data_ptr(), rd.data_ptr(), out.data_ptr(),
                                        lse.data_ptr(), cs.data_ptr(), N, L, C, heads, cross, _s()) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    o64 = out.to(F64).reshape(N, L, 1, C)
    assert_sums(cs.to(F64), G.cstats(o64), G.cstats(o64.abs()), 1e-6, 'attention cstats')
    # chain: two roundings (P and the output) in the tensor-core kernel
    assert rel_l2(out, _attn_ref(qkv, res, heads, cross)) < (1e-2 if dtype == 1 else 2e-5)


# ======================================================================================================================
# apply: gn_apply_vec_kernel<T, FILM> / gn_apply_kernel
# ======================================================================================================================
def _kappa(gs, H, W, C):
    """per-(sample, channel) cancellation ratio of the fp32 variance E[x^2] - mean^2: (E[x^2] + mean^2) / (var + eps)"""
    cnt = G.count(H, W, C)
    m = gs[..., 0] / cnt
    q = gs[..., 1] / cnt
    k = (q + m * m) / (torch.clamp(q - m * m, min=0.) + G.EPS)
    return k[:, G.group_of(C)]


def _rstd_tol(kappa):
    """relative error of the kernels' rstd / -mean*rstd from fp32 group sums: mean = s * inv_cnt and E[x^2] = q * inv_cnt carry
    2 roundings each, mean^2 one more, the difference one: |d var| <= 5 u (E[x^2] + mean^2), so rstd = (var + eps)^-1/2 errs by
    <= 2.5 u kappa, plus rsqrtf (2 ulp) -> 2^-22 kappa + 1e-5 (the 1e-5 the table is held to when nothing cancels)"""
    return 2. ** -22 * kappa + 1e-5


APPLY_CASES = [
    # dtype, N, H, W, C, ca, mode, rs, train, drop_rate, params_out, shift
    (1, 6, 8, 8, 32, 32, G.PLAIN, G.RS_NONE, 0, 0., True, 0.),
    (1, 4, 5, 7, 96, 64, G.SWISH, G.RS_NONE, 0, 0., True, 0.),     # 3 channels per group, concat split inside group 21; 70 px
    (1, 4, 8, 8, 256, 256, G.FILM, G.RS_NONE, 1, 0.3, True, 0.),   # dropout in training
    (1, 4, 6, 6, 768, 512, G.FILM, G.RS_NONE, 0, 0.3, False, 0.),  # 24 channels per group; eval: no dropout
    (1, 4, 8, 8, 1024, 1024, G.SWISH, G.RS_NONE, 0, 0., False, 0.),
    (1, 4, 4, 4, 2048, 2048, G.PLAIN, G.RS_NONE, 0, 0., True, 0.),
    (0, 4, 4, 4, 2048, 1024, G.SWISH, G.RS_NONE, 0, 0., True, 0.),  # fp32: 512 vectors of 4 -> two per thread
    (0, 6, 5, 3, 96, 64, G.FILM, G.RS_NONE, 1, 0.2, True, 0.),
    (1, 4, 8, 8, 64, 64, G.SWISH, G.RS_DOWN, 0, 0., False, 0.),
    (1, 6, 6, 6, 96, 96, G.PLAIN, G.RS_UP, 0, 0., False, 0.),
    (0, 4, 8, 6, 64, 32, G.PLAIN, G.RS_DOWN, 0, 0., False, 0.),
    (0, 4, 4, 4, 64, 64, G.SWISH, G.RS_UP, 0, 0., False, 0.),
    (1, 4, 8, 8, 128, 128, G.SWISH, G.RS_NONE, 0, 0., True, 30.),  # |mean| / sigma ~ 25
]


def _apply_inputs(case):
    dtype, N, H, W, C, ca, mode, rs, train, rate, pout, shift = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFFFF)
    # per-sample and per-group offsets and scales: statistics that differ by sample, group and frame
    smp = torch.arange(N, device='cuda', dtype=F64)[:, None, None, None]
    grp = G.group_of(C).to('cuda', F64)
    x = _q(_rand((N, H, W, C), g, 1.) * (1. + 0.02 * grp) + 0.3 * smp + 0.05 * grp + shift, dtype)
    gamma = (1. + 0.3 * torch.randn(C, generator=g, dtype=F64)).float().cuda()
    beta = (0.2 * torch.randn(C, generator=g, dtype=F64)).float().cuda()
    e = _q(_rand((N, H, W, 2 * C), g, 0.5), dtype) if mode == G.FILM else None
    return x, gamma, beta, e


def _run_apply(lib, case, x, gamma, beta, e, cs):
    dtype, N, H, W, C, ca, mode, rs, train, rate, pout, shift = case
    Ho, Wo = (H // 2, W // 2) if rs == G.RS_DOWN else ((2 * H, 2 * W) if rs == G.RS_UP else (H, W))
    y = torch.zeros(N, Ho, Wo, C, dtype=DT[dtype], device='cuda')
    stats = torch.zeros(N // 2, 32, 2, dtype=torch.float32, device='cuda')
    params = torch.zeros(N // 2, C, 4, dtype=torch.float32, device='cuda') if pout else None
    csa, csb = cs[:, :ca].contiguous(), cs[:, ca:].contiguous()
    seed = _seed_dev()
    xd, ed = _dev(x, dtype), _dev(e, dtype)
    rc = lib.xunet_op_groupnorm(dtype, xd.data_ptr(), csa.data_ptr(), csb.data_ptr() if ca < C else None, ca,
                                gamma.data_ptr(), beta.data_ptr(), _p(ed),
                                y.data_ptr(), stats.data_ptr(), params.data_ptr() if pout else None, N, H, W, C, mode, rs, rate,
                                5, seed.data_ptr(), train, _s())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    return y, stats, params


@pytest.mark.parametrize('case', APPLY_CASES)
def test_groupnorm_apply(lib, case):
    dtype, N, H, W, C, ca, mode, rs, train, rate, pout, shift = case
    x, gamma, beta, e = _apply_inputs(case)
    cs = G.cstats(x).float()                    # the producer's statistics: the kernel's input
    y, stats, params = _run_apply(lib, case, x, gamma, beta, e, cs)
    cs64 = cs.to(F64)
    # group sums: fp32 adds of C/32 channel sums in a fixed tree, <= 5 u sum|terms|
    assert_sums(stats.to(F64), G.group_sums(cs64), G.group_sums(cs64.abs()), 1e-6, 'stats')
    gs = G.group_sums(cs64)
    mean, rstd = G.mean_rstd_from_sums(gs, H, W, C)
    tol = _rstd_tol(_kappa(gs, H, W, C))
    if pout:
        t = G.table(mean, rstd, gamma, beta)
        assert_elems(params[..., :2], t[..., :2], 0., tol[..., None], 'table {rstd, -mean*rstd}')
        assert torch.equal(params[..., 2:].to(F64), t[..., 2:]), 'table {gamma, beta}'
    keep = torch.from_numpy(keep_mask(SEED, 5, (N, H, W, C), rate)).cuda() if (mode == G.FILM and train and rate > 0) else None
    ref = G.forward(x, gamma.to(F64), beta.to(F64), mode, rs, e=e, keep=keep, drop_rate=rate, mean=mean, rstd=rstd)
    # floor: yhat = x * (rstd gamma) + (beta - mean rstd gamma) in fp32 errs by tol |xhat gamma| through rstd and by
    # 2^-22 (|x rstd gamma| + |mean rstd gamma| + |beta|) through the two fmas; swish' <= 1.1, FiLM scales it by |1 + scale|
    # and the keep scale
    xh = G.xhat(x, mean, rstd)
    m_b, r_b = (G._per_channel(t, N, H, W) for t in (mean, rstd))
    gm, bt = gamma.to(F64), beta.to(F64)
    fl = (G._per_channel(tol, N, H, W) * (xh * gm).abs() + 2. ** -22 * ((x * r_b * gm).abs() + (m_b * r_b * gm).abs() + bt.abs()))
    if mode != G.PLAIN:
        fl = fl * 1.1
    if mode == G.FILM:
        fl = fl * (1. + e[..., :C]).abs() + 2. ** -22 * e[..., C:].abs()
        if keep is not None:
            fl = fl * G.keep_scale(rate)
    fl = G.resample(fl, rs)
    assert_elems(y, ref, fl, BF_REL if dtype == 1 else F32_REL, 'y')
    # chain: the exact two-pass statistics of x
    ref_exact = G.forward(x, gamma.to(F64), beta.to(F64), mode, rs, e=e, keep=keep, drop_rate=rate)
    if shift == 0.:
        assert rel_l2(y, ref_exact) < (6e-3 if dtype == 1 else 1e-5)
    else:
        # |mean| / sigma ~ 25-30: kappa = 1 + 2 (mean / sigma)^2 ~ 2000, so the fp32 E[x^2] - mean^2 variance gives rstd to
        # 2^-22 kappa ~ 5e-4 relative at worst (an H100 measured 2e-5), i.e. yhat errs by <= 5e-4 |xhat gamma|: under the
        # bf16 rounding of y.
        em, er = G.mean_rstd(x)
        got_r = params[..., 0].to(F64)
        rstd_err = float(((got_r - er) / er).abs().max())
        print(f'|mean|/sigma ~ {float((em / (1 / er)).abs().mean()):.1f}: kappa max {float(_kappa(gs, H, W, C).max()):.0f}, '
              f'rstd relative error vs two-pass fp64 {rstd_err:.2e}')
        assert rstd_err < float(tol.max())
        assert rel_l2(y, ref_exact) < 6e-3


# ======================================================================================================================
# the consumer conv's data gradient with the norm's first backward pass: EPI 2 (plain / swish) and EPI 3 (FiLM + dropout)
# ======================================================================================================================
EPI2_CASES = [
    # N, H, W, C (norm), Co (consumer), ks, nseg, mode, alpha
    (6, 16, 16, 64, 48, 3, 1, G.SWISH, 1.),          # BK 16, BN 32, two CTAs per SM
    (6, 64, 64, 64, 48, 3, 1, G.SWISH, 0.7071),      # BK 16, BN 64: one CTA per SM; 192 tiles on 132 CTAs
    (6, 64, 64, 128, 128, 3, 1, G.SWISH, 1.),        # BK 32, BN 128, persistent
    (6, 64, 64, 64, 96, 3, 1, G.SWISH, 1.),          # BK 32, BN 64, two CTAs per SM
    (16, 4, 4, 64, 64, 3, 1, G.SWISH, 1.),           # 16-pixel images (no halo), BK 64
    (6, 8, 8, 64, 192, 1, 3, G.PLAIN, 1.),           # the attention norm's q|k|v projection, BN 32
    (12, 64, 64, 64, 192, 1, 3, G.PLAIN, 1.),        # q|k|v, BN 64, two CTAs per SM, 384 tiles on 264 CTAs
]
EPI3_CASES = [
    # N, H, W, C, Co, ks, nseg, drop_rate, train
    (6, 16, 16, 64, 64, 3, 1, 0.3, 1),               # BN 32
    (6, 64, 64, 64, 64, 3, 1, 0.1, 1),               # BN 64, persistent
    (6, 64, 64, 128, 128, 3, 1, 0.3, 0),             # BN 128, no dropout (eval)
    (16, 4, 4, 64, 64, 3, 1, 0.3, 1),                # 16-pixel images
    (6, 32, 32, 32, 32, 3, 1, 0., 1),                # BN 32, BK 32, rate 0
]


def _gn_forward_state(g, N, H, W, C, film):
    """the norm's input x (bf16), gamma, beta, its params table as the forward stores it (fp32), e"""
    smp = torch.arange(N, device='cuda', dtype=F64)[:, None, None, None]
    x = _q(_rand((N, H, W, C), g) * 1.3 + 0.4 * smp + 0.1 * G.group_of(C).to('cuda', F64), 1)
    gamma = (1. + 0.3 * torch.randn(C, generator=g, dtype=F64)).float().cuda()
    beta = (0.2 * torch.randn(C, generator=g, dtype=F64)).float().cuda()
    mean, rstd = G.mean_rstd(x)
    table = G.table(mean, rstd, gamma, beta).float().contiguous()
    e = _q(_rand((N, H, W, 2 * C), g, 0.5), 1) if film else None
    return x, gamma, beta, table, e


def _run_epi(lib, g, N, H, W, C, Co, ks, nseg, mode, alpha, rate=0., train=0):
    taps = ks * ks
    x, gamma, beta, table, e = _gn_forward_state(g, N, H, W, C, mode == G.FILM)
    w = _rand((taps, C, Co), g, 1 / math.sqrt(taps * Co)).float()
    dy = _q(_rand((N, H, W, Co), g), 1)
    dyh = torch.zeros(N, H, W, C, dtype=torch.bfloat16, device='cuda')
    de = torch.zeros(N, H, W, 2 * C, dtype=torch.bfloat16, device='cuda') if mode == G.FILM else None
    bcs = torch.zeros(N // 2, C, 2, dtype=torch.float32, device='cuda')
    seed = _seed_dev()
    dyd, xd, ed = _dev(dy, 1), _dev(x, 1), _dev(e, 1)
    rc = lib.xunet_op_conv_dgrad_groupnorm(1, dyd.data_ptr(), w.data_ptr(), xd.data_ptr(), table.data_ptr(), mode, _p(ed),
                                           de.data_ptr() if de is not None else None, rate, 7, seed.data_ptr(), train,
                                           dyh.data_ptr(), bcs.data_ptr(), N, H, W, C, Co, ks, nseg, alpha, _s())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    return dict(x=x, gamma=gamma, beta=beta, table=table, e=e, w=w, dy=dy, dyh=dyh, de=de, bcs=bcs)


def _check_epi(r, N, H, W, C, Co, ks, nseg, mode, alpha, rate=0., train=0):
    x, table, e = r['x'], r['table'].to(F64), r['e']
    wb = r['w'].to(torch.bfloat16).to(F64)
    gact = alpha * _dgrad_ref(r['dy'], wb, ks, C, nseg)
    gmag = alpha * _dgrad_ref(r['dy'].abs(), wb.abs(), ks, C, nseg) * CONV_FLOOR(ks * ks * Co)   # the floor of the conv's sum
    # stage: dyhat from the kernel's inputs, the norm taken from the stored table (xhat = x rstd + (-mean rstd))
    rstd, nmr = table[..., 0], table[..., 1]
    mean = -nmr / rstd
    keep = torch.from_numpy(keep_mask(SEED, 7, (N, H, W, C), rate)).cuda() if (mode == G.FILM and train and rate > 0) else None
    dyh_ref, de_ref = G.dyhat(gact, x, table[..., 2][0], table[..., 3][0], mode, e=e, keep=keep, drop_rate=rate, mean=mean,
                              rstd=rstd)
    # floor: the conv's accumulation (gmag: CONV_FLOOR of its terms) times the local derivative (<= 1.1 for swish; FiLM: also
    # |1 + scale| and the keep scale), plus the fp32 evaluation of the derivative's argument (2^-21 of its terms, times
    # |g| max|swish''| <= 0.5)
    xh = G.xhat(x, mean, rstd)
    gm, bt = table[0, :, 2], table[0, :, 3]
    yh = xh * gm + bt
    yterms = (x * G._per_channel(rstd, N, H, W) * gm).abs() + (G._per_channel(nmr, N, H, W) * gm).abs() + bt.abs()
    if mode == G.PLAIN:
        fl = gmag
    elif mode == G.SWISH:
        fl = 1.1 * gmag + 0.5 * 2. ** -21 * gact.abs() * yterms
    else:
        sc, sh = e[..., :C], e[..., C:]
        ks_ = G.keep_scale(rate) if keep is not None else 1.
        uterms = yterms * (1. + sc).abs() + sh.abs()
        fl_du = ks_ * (1.1 * gmag + 0.5 * 2. ** -21 * gact.abs() * uterms)
        fl = fl_du * (1. + sc).abs()
        du = de_ref[..., C:]
        assert_elems(r['de'], de_ref, torch.cat([fl_du * yh.abs() + du.abs() * 2. ** -21 * yterms, fl_du], -1), BF_REL,
                     'de = [du*yhat | du]')
    assert_elems(r['dyh'], dyh_ref, fl, BF_REL, 'dyhat')
    # bcs: the channel sums of the STORED dyhat times xhat, in fp64.  The epilogue forms xhat in fp32 (2^-22 relative of
    # |x rstd| + |mean rstd|) and sums 32-row slices in fp32 (<= 2^-19), the slices in fp64: 1e-5 sum|terms|.
    d = r['dyh'].to(F64)
    ref = G.bcs(d, xh)
    xh_terms = (x * G._per_channel(rstd, N, H, W)).abs() + G._per_channel(nmr, N, H, W).abs()
    terms = torch.stack([G.bcs(d.abs(), xh_terms)[..., 0], G.bcs(d.abs(), xh_terms)[..., 1]], -1)
    assert_sums(r['bcs'].to(F64), ref, terms, 1e-5, 'bcs')
    # chain: dyhat from the bf16 inputs and the exact statistics of x (one rounding: the stored dyhat)
    dyh_exact, _ = G.dyhat(gact, x, r['gamma'].to(F64), r['beta'].to(F64), mode, e=e, keep=keep, drop_rate=rate)
    assert rel_l2(r['dyh'], dyh_exact) < 6e-3


@pytest.mark.parametrize('case', EPI2_CASES)
def test_conv_dgrad_groupnorm_epi2(lib, case):
    N, H, W, C, Co, ks, nseg, mode, alpha = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFFFF)
    r = _run_epi(lib, g, N, H, W, C, Co, ks, nseg, mode, alpha)
    _check_epi(r, N, H, W, C, Co, ks, nseg, mode, alpha)


@pytest.mark.parametrize('case', EPI3_CASES)
def test_conv_dgrad_groupnorm_epi3(lib, case):
    N, H, W, C, Co, ks, nseg, rate, train = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFFFF)
    r = _run_epi(lib, g, N, H, W, C, Co, ks, nseg, G.FILM, 1., rate, train)
    _check_epi(r, N, H, W, C, Co, ks, nseg, G.FILM, 1., rate, train)


# ======================================================================================================================
# backward apply: gn_bwd_apply_pre_kernel (fused path) and gn_bwd_reduce_kernel + gn_bwd_apply_kernel
# ======================================================================================================================
def _dx_floor(dyh, xh, mean, rstd, gamma, sums, extra_term, old):
    """floor of dx = rstd (gamma dyhat - S1/cnt - xhat S2/cnt) evaluated in fp32 as dyhat kg + x kx + k0 (or with xhat formed
    first): every term is rounded a few times (2^-21 of it), rstd enters squared through kx (2 x the rstd error), S1 / S2 are
    fp32 sums of gamma * channel sums (2^-21 of sum |gamma sums|); x kx and k0 cancel to xhat S2, so the x-term counts
    |xhat| + |mean rstd|"""
    N, H, W, C = dyh.shape
    cnt = G.count(H, W, C)
    B = N // 2
    s1a = (gamma.abs() * sums[..., 1].abs()).reshape(B, 32, -1).sum(-1)[:, G.group_of(C)] / cnt
    s2a = (gamma.abs() * sums[..., 0].abs()).reshape(B, 32, -1).sum(-1)[:, G.group_of(C)] / cnt
    r = G._per_channel(rstd, N, H, W)
    mr = G._per_channel((mean * rstd).abs(), N, H, W)
    terms = r * ((gamma * dyh).abs() + G._per_channel(s1a, N, H, W) + (xh.abs() + mr) * G._per_channel(s2a, N, H, W))
    return 2. ** -19 * terms + 2. ** -22 * (extra_term + old)


BWD_PRE_CASES = [
    # dtype, N, H, W, C, extra, accumulate
    (1, 6, 16, 16, 64, True, False),
    (1, 4, 8, 8, 256, False, True),
    (1, 4, 5, 7, 96, True, True),
    (0, 4, 8, 8, 2048, True, False),
    (0, 6, 4, 6, 64, False, True),
]


@pytest.mark.parametrize('case', BWD_PRE_CASES)
def test_groupnorm_bwd_fused(lib, case):
    dtype, N, H, W, C, has_extra, acc = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFFFF)
    smp = torch.arange(N, device='cuda', dtype=F64)[:, None, None, None]
    x = _q(_rand((N, H, W, C), g) + 0.3 * smp, dtype)
    gamma = (1. + 0.3 * torch.randn(C, generator=g, dtype=F64)).float().cuda()
    beta = (0.2 * torch.randn(C, generator=g, dtype=F64)).float().cuda()
    dyh = _q(_rand((N, H, W, C), g), dtype)
    stats = G.group_sums(G.cstats(x)).float()
    mean, rstd = G.mean_rstd_from_sums(stats.to(F64), H, W, C)
    xh = G.xhat(x, mean, rstd)
    bcs = G.bcs(dyh, xh).float()                           # what the epilogue emitted (the kernel's input)
    extra = _q(_rand((N, H, W, C), g), dtype) if has_extra else None
    old = _q(_rand((N, H, W, C), g), dtype) if acc else torch.zeros(N, H, W, C, dtype=F64, device='cuda')
    dx = _dev(old, dtype)
    dg0 = _rand((C,), g).float()
    db0 = _rand((C,), g).float()
    dgamma, dbeta = dg0.clone(), db0.clone()
    ea = 0.7071
    xd, gd, exd = _dev(x, dtype), _dev(dyh, dtype), _dev(extra, dtype)
    rc = lib.xunet_op_groupnorm_bwd(dtype, xd.data_ptr(), None, gd.data_ptr(), dx.data_ptr(), None,
                                    gamma.data_ptr(), beta.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), stats.data_ptr(), None,
                                    bcs.data_ptr(), _p(exd), ea, N, H, W, C,
                                    G.SWISH, G.RS_NONE, 0., 0, None, 1, int(acc), 0, _s())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    b64 = bcs.to(F64)
    ref, _ = G.dx(dyh, xh, rstd, gamma.to(F64), b64)
    et = (ea * extra).abs() if has_extra else 0.
    if has_extra:
        ref = ref + ea * extra
    ref = ref + old
    fl = _dx_floor(dyh, xh, mean, rstd, gamma.to(F64), b64, et, old.abs())
    assert_elems(dx, ref, fl, BF_REL if dtype == 1 else F32_REL, 'dx')
    # dgamma / dbeta: one block adds the samples' channel sums in sample order in fp32, then adds that to the initial value
    ga = torch.zeros(C, dtype=torch.float32, device='cuda')
    gb = torch.zeros(C, dtype=torch.float32, device='cuda')
    for b in range(N // 2):
        ga, gb = ga + bcs[b, :, 0], gb + bcs[b, :, 1]
    assert torch.equal(dgamma, dg0 + ga) and torch.equal(dbeta, db0 + gb), 'dgamma / dbeta'


BWD_CASES = [
    # dtype, N, H, W, C, mode, rs, drop_rate, train, extra, accumulate, de_accumulate
    (1, 4, 8, 8, 64, G.PLAIN, G.RS_NONE, 0., 0, True, False, False),
    (1, 6, 5, 7, 96, G.SWISH, G.RS_NONE, 0., 0, False, True, False),
    (1, 4, 8, 8, 128, G.FILM, G.RS_NONE, 0.3, 1, False, False, True),
    (0, 4, 6, 6, 64, G.FILM, G.RS_NONE, 0.3, 0, True, False, False),
    (1, 4, 8, 8, 64, G.SWISH, G.RS_DOWN, 0., 0, False, False, False),
    (1, 4, 6, 6, 64, G.PLAIN, G.RS_UP, 0., 0, False, True, False),
    (0, 4, 4, 6, 96, G.SWISH, G.RS_DOWN, 0., 0, False, True, False),
    (0, 4, 4, 4, 2048, G.SWISH, G.RS_UP, 0., 0, False, False, False),
]


@pytest.mark.parametrize('case', BWD_CASES)
def test_groupnorm_bwd_two_kernel(lib, case):
    dtype, N, H, W, C, mode, rs, rate, train, has_extra, acc, de_acc = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFFFF)
    smp = torch.arange(N, device='cuda', dtype=F64)[:, None, None, None]
    x = _q(_rand((N, H, W, C), g) + 0.3 * smp, dtype)
    gamma = (1. + 0.3 * torch.randn(C, generator=g, dtype=F64)).float().cuda()
    beta = (0.2 * torch.randn(C, generator=g, dtype=F64)).float().cuda()
    e = _q(_rand((N, H, W, 2 * C), g, 0.5), dtype) if mode == G.FILM else None
    Ho, Wo = (H // 2, W // 2) if rs == G.RS_DOWN else ((2 * H, 2 * W) if rs == G.RS_UP else (H, W))
    dout = _q(_rand((N, Ho, Wo, C), g), dtype)
    stats = G.group_sums(G.cstats(x)).float()
    mean, rstd = G.mean_rstd_from_sums(stats.to(F64), H, W, C)
    extra = _q(_rand((N, H, W, C), g), dtype) if has_extra else None
    old = _q(_rand((N, H, W, C), g), dtype) if acc else torch.zeros(N, H, W, C, dtype=F64, device='cuda')
    de_old = _q(_rand((N, H, W, 2 * C), g), dtype) if de_acc else torch.zeros(N, H, W, 2 * C, dtype=F64, device='cuda')
    dx, de = _dev(old, dtype), _dev(de_old, dtype)
    dg0, db0 = _rand((C,), g).float(), _rand((C,), g).float()
    dgamma, dbeta = dg0.clone(), db0.clone()
    bstats = torch.full((N // 2, 32, 2), 7., dtype=torch.float32, device='cuda')    # an output: overwritten
    seed = _seed_dev()
    ea = 0.7071
    xd, ed, gd, exd = _dev(x, dtype), _dev(e, dtype), _dev(dout, dtype), _dev(extra, dtype)
    rc = lib.xunet_op_groupnorm_bwd(dtype, xd.data_ptr(), _p(ed), gd.data_ptr(), dx.data_ptr(), de.data_ptr() if e is not None else None,
                                    gamma.data_ptr(), beta.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), stats.data_ptr(),
                                    bstats.data_ptr(), None, _p(exd), ea, N, H, W, C,
                                    mode, rs, rate, 9, seed.data_ptr(), train, int(acc), int(de_acc), _s())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    gm64 = gamma.to(F64)
    keep = torch.from_numpy(keep_mask(SEED, 9, (N, H, W, C), rate)).cuda() if (mode == G.FILM and train and rate > 0) else None
    xh = G.xhat(x, mean, rstd)
    dyh, de_ref = G.dyhat(G.resample_adjoint(dout, rs), x, gm64, beta.to(F64), mode, e=e, keep=keep, drop_rate=rate, mean=mean,
                          rstd=rstd)
    sums = G.bcs(dyh, xh)
    abs_sums = G.bcs(dyh.abs(), xh.abs())
    # sums over pixels: fp32 per thread (a few hundred terms at most, <= 2^-16), fp64 across threads and blocks: 1e-5 sum|terms|
    # (the fp32 dyhat itself errs by ~2^-21 of its terms)
    assert_sums(dgamma.to(F64), dg0.to(F64) + sums[..., 0].sum(0), abs_sums[..., 0].sum(0) + dg0.to(F64).abs() * 1e-2, 1e-5,
                'dgamma')
    assert_sums(dbeta.to(F64), db0.to(F64) + sums[..., 1].sum(0), abs_sums[..., 1].sum(0) + db0.to(F64).abs() * 1e-2, 1e-5,
                'dbeta')
    assert_sums(bstats.to(F64), G.group_bsums(gm64, sums), G.group_bsums(gm64.abs(), abs_sums), 1e-5, 'bstats [S1, S2]')
    ref, _ = G.dx(dyh, xh, rstd, gm64, sums)
    et = (ea * extra).abs() if has_extra else 0.
    if has_extra:
        ref = ref + ea * extra
    ref = ref + old
    assert_elems(dx, ref, _dx_floor(dyh, xh, mean, rstd, gm64, sums, et, old.abs()), BF_REL if dtype == 1 else F32_REL, 'dx')
    if mode == G.FILM:
        # de = [du yhat | du] (+ the old value): du from fp32 u and swish'(u): 2^-20 of |g| (1 + |u terms|) as in the EPI 3 check
        yh = xh * gm64 + beta.to(F64)
        sc, sh = e[..., :C], e[..., C:]
        gk = dout * (keep.to(F64) * G.keep_scale(rate) if keep is not None else 1.)
        fl_du = 2. ** -20 * gk.abs() * (1. + (yh * (1. + sc)).abs() + sh.abs() + (xh * gm64).abs() + beta.to(F64).abs())
        fl = torch.cat([fl_du * (1. + yh.abs()), fl_du], -1) + 2. ** -22 * de_old.abs()
        assert_elems(de, de_ref + de_old, fl, BF_REL if dtype == 1 else F32_REL, 'de')


def test_fused_backward_chain_from_bf16_inputs(lib):
    """EPI 2 then the fused apply, against the fp64 backward of the bf16 inputs with exact statistics: two roundings (the
    stored dyhat and dx)"""
    N, H, W, C, Co, ks = 6, 16, 16, 64, 96, 3
    g = torch.Generator().manual_seed(77)
    r = _run_epi(lib, g, N, H, W, C, Co, ks, 1, G.SWISH, 1.)
    x, gamma, beta = r['x'], r['gamma'], r['beta']
    stats = G.group_sums(G.cstats(x)).float()
    dx = torch.zeros(N, H, W, C, dtype=torch.bfloat16, device='cuda')
    dgamma = torch.zeros(C, dtype=torch.float32, device='cuda')
    dbeta = torch.zeros(C, dtype=torch.float32, device='cuda')
    xd = _dev(x, 1)
    assert lib.xunet_op_groupnorm_bwd(1, xd.data_ptr(), None, r['dyh'].data_ptr(), dx.data_ptr(), None, gamma.data_ptr(),
                                      beta.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), stats.data_ptr(), None,
                                      r['bcs'].data_ptr(), None, 0., N, H, W, C, G.SWISH, G.RS_NONE, 0., 0, None, 1, 0, 0,
                                      _s()) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    wb = r['w'].to(torch.bfloat16).to(F64)
    gact = _dgrad_ref(r['dy'], wb, ks, C)
    mean, rstd = G.mean_rstd(x)
    dyh, _ = G.dyhat(gact, x, gamma.to(F64), beta.to(F64), G.SWISH)
    xh = G.xhat(x, mean, rstd)
    sums = G.bcs(dyh, xh)
    ref, _ = G.dx(dyh, xh, rstd, gamma.to(F64), sums)
    assert rel_l2(dx, ref) < 1e-2
    assert rel_l2(dgamma, sums[..., 0].sum(0)) < 6e-3 and rel_l2(dbeta, sums[..., 1].sum(0)) < 6e-3


# ======================================================================================================================
# argument checks: every entry returns non-zero with a message before launching anything
# ======================================================================================================================
def test_entry_point_errors(lib):
    t = torch.zeros(1 << 16, dtype=torch.float32, device='cuda')
    p = t.data_ptr()
    s = _s()

    def bad(rc, what):
        assert rc != 0, what
        assert lib.xunet_last_error(), what

    # conv statistics: NULL cstats, C % 32, ksize, an unsupported tensor-core shape
    bad(lib.xunet_op_conv_stats(1, 1, p, p, p, None, p, None, 2, 8, 8, 32, 64, 3, 1., s), 'conv_stats NULL cstats')
    bad(lib.xunet_op_conv_stats(1, 1, p, p, p, None, p, p, 2, 8, 8, 32, 48, 3, 1., s), 'conv_stats C % 32')
    bad(lib.xunet_op_conv_stats(1, 1, p, p, p, None, p, p, 2, 8, 8, 32, 64, 5, 1., s), 'conv_stats ksize')
    bad(lib.xunet_op_conv_stats(1, 1, p, p, p, None, p, p, 3, 8, 8, 32, 64, 3, 1., s), 'conv_stats odd N')
    bad(lib.xunet_op_conv_stats(0, 1, p, p, p, None, p, p, 2, 8, 8, 32, 64, 3, 1., s), 'conv_stats fp32 on tensor cores')
    # attention statistics
    bad(lib.xunet_op_attention_stats(1, 1, p, p, p, p, None, 2, 128, 64, 2, 0, s), 'attention_stats NULL cstats')
    bad(lib.xunet_op_attention_stats(1, 1, p, p, p, p, p, 2, 128, 48, 2, 0, s), 'attention_stats C % 32')
    bad(lib.xunet_op_attention_stats(1, 1, p, p, p, p, p, 2, 100, 64, 2, 0, s), 'attention_stats tensor-core L')
    # apply
    gnp = lambda **k: dict(dtype=1, x=p, ca_=p, cb=None, ca=64, gamma=p, beta=p, e=None, y=p, stats=p, pout=None, N=2, H=8, W=8,
                           C=64, mode=G.SWISH, rs=G.RS_NONE, rate=0., op=0, seed=None, train=0) | k
    def gn(**k):
        a = gnp(**k)
        return lib.xunet_op_groupnorm(a['dtype'], a['x'], a['ca_'], a['cb'], a['ca'], a['gamma'], a['beta'], a['e'], a['y'],
                                      a['stats'], a['pout'], a['N'], a['H'], a['W'], a['C'], a['mode'], a['rs'], a['rate'], a['op'],
                                      a['seed'], a['train'], s)
    bad(gn(C=48, ca=48), 'groupnorm C % 32')
    bad(gn(x=None), 'groupnorm NULL x')
    bad(gn(ca=32), 'groupnorm split without cstats_b')
    bad(gn(ca=0), 'groupnorm ca = 0')
    bad(gn(mode=G.FILM, e=p, rs=G.RS_DOWN), 'groupnorm FiLM on a resampling norm')
    bad(gn(rs=G.RS_UP, pout=p), 'groupnorm params_out on a resampling norm')
    bad(gn(mode=G.FILM), 'groupnorm FiLM without e')
    bad(gn(mode=G.FILM, e=p, rate=0.1, train=1), 'groupnorm dropout without seed')
    bad(gn(rate=1.), 'groupnorm drop_rate 1')
    bad(gn(mode=3), 'groupnorm mode')
    bad(gn(rs=G.RS_DOWN, H=7), 'groupnorm RS_DOWN odd H')
    bad(gn(dtype=2), 'groupnorm dtype')

    # fused data gradient: unsupported shapes (12x12 images do not tile; 8-pixel images put two samples in a warp's rows)
    def dg(**k):
        a = dict(dtype=1, dy=p, w=p, x=p, par=p, mode=G.SWISH, e=None, de=None, rate=0., seed=None, train=0, dyh=p, bcs=p, N=2,
                 H=8, W=8, C=64, Co=64, ks=3, nseg=1) | k
        return lib.xunet_op_conv_dgrad_groupnorm(a['dtype'], a['dy'], a['w'], a['x'], a['par'], a['mode'], a['e'], a['de'],
                                                 a['rate'], 0, a['seed'], a['train'], a['dyh'], a['bcs'], a['N'], a['H'], a['W'],
                                                 a['C'], a['Co'], a['ks'], a['nseg'], 1., s)
    bad(dg(H=12, W=12), 'dgrad_groupnorm untileable shape')
    bad(dg(N=16, H=2, W=4), 'dgrad_groupnorm 8-pixel images')
    bad(dg(bcs=None), 'dgrad_groupnorm NULL bcs')
    bad(dg(C=48), 'dgrad_groupnorm C % 32')
    bad(dg(mode=G.FILM), 'dgrad_groupnorm FiLM without e')
    bad(dg(mode=G.FILM, e=p), 'dgrad_groupnorm FiLM without de')
    bad(dg(e=p), 'dgrad_groupnorm e on a swish norm')
    bad(dg(dtype=0), 'dgrad_groupnorm fp32')
    bad(dg(ks=1, Co=64, nseg=3), 'dgrad_groupnorm Co % nseg')

    # backward apply
    def bw(**k):
        a = dict(dtype=1, x=p, e=None, dy=p, dx=p, de=None, gamma=p, beta=p, dg=p, db=p, stats=p, bstats=p, bcs=None, extra=None,
                 N=2, H=8, W=8, C=64, mode=G.SWISH, rs=G.RS_NONE, rate=0., seed=None, train=0) | k
        return lib.xunet_op_groupnorm_bwd(a['dtype'], a['x'], a['e'], a['dy'], a['dx'], a['de'], a['gamma'], a['beta'], a['dg'],
                                          a['db'], a['stats'], a['bstats'], a['bcs'], a['extra'], 0., a['N'], a['H'], a['W'],
                                          a['C'], a['mode'], a['rs'], a['rate'], 0, a['seed'], a['train'], 0, 0, s)
    bad(bw(C=40), 'groupnorm_bwd C % 32')
    bad(bw(bcs=p, rs=G.RS_DOWN), 'groupnorm_bwd fused with resampling')
    bad(bw(bstats=None), 'groupnorm_bwd two-kernel without bstats')
    bad(bw(mode=G.FILM, e=p), 'groupnorm_bwd FiLM without de')
    bad(bw(mode=G.FILM, rs=G.RS_UP, e=p, de=p), 'groupnorm_bwd FiLM with resampling')
    bad(bw(dg=None), 'groupnorm_bwd NULL dgamma')
    torch.cuda.synchronize()
    assert bool((t == 0).all()), 'a rejected call launched a kernel'


# ======================================================================================================================
# coverage of the conv epilogue variants, read from the launcher's log in a child process (the flag is read once per process)
# ======================================================================================================================
# (epi, BN, bk, halo, per_sm) every case list above is meant to reach
REQUIRED_VARIANTS = {
    (1, 32, 32, 1, 2), (1, 32, 32, 0, 2), (1, 32, 64, 0, 2), (1, 64, 32, 1, 2), (1, 128, 32, 1, 1),
    (2, 32, 16, 1, 2), (2, 64, 16, 1, 1), (2, 128, 32, 1, 1), (2, 64, 32, 1, 2), (2, 32, 64, 0, 2), (2, 64, 64, 0, 2),
    (3, 32, 64, 1, 1), (3, 64, 64, 1, 1), (3, 128, 32, 1, 1), (3, 32, 64, 0, 1), (3, 32, 32, 1, 1),
}


def test_conv_epilogue_variants_reached(lib):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, XUNET_CONV_LOG='1')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-s', '-p', 'no:cacheprovider', '-m', 'gpu',
                        os.path.join(root, 'tests', 'test_gpu_groupnorm.py'), '-k', 'conv_stats or epi2 or epi3'],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    seen, multi = set(), set()
    for line in r.stderr.splitlines():
        if not line.startswith('conv_tc mode='):
            continue
        kv = dict(re.findall(r'(\w+)=(-?\d+)', line))
        key = (int(kv['epi']), int(kv['BN']), int(kv['bk']), int(kv['halo']), int(kv['per_sm']))
        seen.add(key)
        if key[0] >= 2 and int(kv['tiles']) > int(kv['ctas']):     # a persistent grid: some CTAs take several tiles
            multi.add(key)
    print('conv epilogue variants seen (epi, BN, bk, halo, per_sm):', sorted(seen))
    print('fused-backward variants with more tiles than CTAs:', sorted(multi))
    assert REQUIRED_VARIANTS <= seen, sorted(REQUIRED_VARIANTS - seen)
    assert any(k[4] == 1 for k in multi) and any(k[4] == 2 for k in multi), multi
