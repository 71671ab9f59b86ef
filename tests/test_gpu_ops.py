"""GPU parity of single kernels through the C-ABI operator entry points, against plain torch-CPU fp64 restatements."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import xunet_ref as R
from tests.util import rel_l2

pytestmark = pytest.mark.gpu

DT = {0: torch.float32, 1: torch.bfloat16}
TOL = {0: 2e-5, 1: 1.5e-2}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ref_conv(x, w, bias, stride, ks):
    """x (N,H,W,Ci) fp64, w (taps,Ci,Co) -> (N,Ho,Wo,Co)  (Flax SAME padding)."""
    N, H, W, Ci = x.shape
    Co = w.shape[-1]
    if ks == 1:
        return x @ w[0] + bias
    k5 = w.reshape(1, 3, 3, Ci, Co)
    y = R.conv_1x3x3(x.reshape(N // 2, 2, H, W, Ci), k5, bias, stride=stride)
    return y.reshape(N, y.shape[2], y.shape[3], Co)


CONV_CASES = [
    # N, H, W, Ci, Co, ks, stride
    (2, 16, 16, 32, 32, 3, 1), (2, 16, 16, 96, 64, 3, 1), (2, 8, 8, 3, 32, 3, 1), (2, 8, 8, 32, 3, 3, 1),
    (2, 16, 16, 144, 32, 3, 2), (2, 16, 16, 144, 32, 3, 4), (2, 16, 16, 144, 32, 3, 8), (4, 8, 8, 64, 128, 1, 1),
    (2, 12, 20, 32, 64, 3, 1), (2, 32, 32, 64, 64, 3, 1),
]


@pytest.mark.parametrize('dtype', [0, 1])
@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_fwd_dgrad_wgrad(lib, dtype, case):
    N, H, W, Ci, Co, ks, stride = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    taps = ks * ks
    x = torch.randn(N, H, W, Ci, generator=g, dtype=torch.float64)
    w = torch.randn(taps, Ci, Co, generator=g, dtype=torch.float64) / math.sqrt(taps * Ci)
    b = torch.randn(Co, generator=g, dtype=torch.float64) * 0.1
    xq = x.to(DT[dtype]).double()           # the oracle sees the same (possibly bf16-rounded) activations
    xr = xq.clone().requires_grad_(True)
    wr = w.float().double().requires_grad_(True)
    br = b.float().double().requires_grad_(True)
    y_ref = _ref_conv(xr, wr, br, stride, ks)
    res = torch.randn(y_ref.shape, generator=g, dtype=torch.float64).to(DT[dtype]).double()
    alpha = 0.7071
    out_ref = (y_ref + res) * alpha
    dy = torch.randn(y_ref.shape, generator=g, dtype=torch.float64).to(DT[dtype]).double()
    out_ref.backward(dy)

    xd = xq.to(DT[dtype]).cuda().contiguous()
    wd, bd = w.float().cuda().contiguous(), b.float().cuda().contiguous()
    resd = res.to(DT[dtype]).cuda().contiguous()
    yd = torch.zeros(y_ref.shape, dtype=DT[dtype], device='cuda')
    assert lib.xunet_op_conv(dtype, 0, xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), resd.data_ptr(), yd.data_ptr(),
                             N, H, W, Ci, Co, ks, stride, 1, alpha, _stream()) == 0, lib.xunet_last_error()
    assert rel_l2(yd.float(), out_ref.detach()) < TOL[dtype]

    dyd = dy.to(DT[dtype]).cuda().contiguous()
    dxd = torch.zeros(x.shape, dtype=DT[dtype], device='cuda')
    assert lib.xunet_op_conv_dgrad(dtype, 0, dyd.data_ptr(), wd.data_ptr(), dxd.data_ptr(), N, H, W, Ci, Co, ks, stride, 1,
                                   alpha, 0, _stream()) == 0, lib.xunet_last_error()
    assert rel_l2(dxd.float(), xr.grad) < TOL[dtype]
    # accumulate flag
    assert lib.xunet_op_conv_dgrad(dtype, 0, dyd.data_ptr(), wd.data_ptr(), dxd.data_ptr(), N, H, W, Ci, Co, ks, stride, 1,
                                   alpha, 1, _stream()) == 0
    assert rel_l2(dxd.float(), 2 * xr.grad) < 2 * TOL[dtype]

    dwd = torch.zeros(taps, Ci, Co, dtype=torch.float32, device='cuda')
    dbd = torch.zeros(Co, dtype=torch.float32, device='cuda')
    assert lib.xunet_op_conv_wgrad(dtype, 0, xd.data_ptr(), dyd.data_ptr(), dwd.data_ptr(), dbd.data_ptr(), N, H, W, Ci, Co,
                                   ks, stride, 1, alpha, _stream()) == 0, lib.xunet_last_error()
    assert rel_l2(dwd, wr.grad) < TOL[dtype]
    assert rel_l2(dbd, br.grad) < TOL[dtype]


@pytest.mark.parametrize('dtype', [0, 1])
def test_fused_qkv_projection_segments(lib, dtype):
    """q|k|v weights are three adjacent (C, heads, hd) Flax leaves read as one (C, 3C) GEMM (nseg=3)."""
    N, H, W, Cc = 2, 8, 8, 64
    g = torch.Generator().manual_seed(11)
    x = torch.randn(N, H, W, Cc, generator=g, dtype=torch.float64).to(DT[dtype]).double()
    ws = [torch.randn(Cc, Cc, generator=g, dtype=torch.float64) / 8 for _ in range(3)]
    bs = [torch.randn(Cc, generator=g, dtype=torch.float64) * 0.1 for _ in range(3)]
    wflat = torch.cat([w.reshape(-1) for w in ws]).float().cuda()
    bflat = torch.cat(bs).float().cuda()
    y = torch.zeros(N, H, W, 3 * Cc, dtype=DT[dtype], device='cuda')
    xd = x.to(DT[dtype]).cuda()
    assert lib.xunet_op_conv(dtype, 0, xd.data_ptr(), wflat.data_ptr(), bflat.data_ptr(), None, y.data_ptr(), N, H, W, Cc,
                             3 * Cc, 1, 1, 3, 1.0, _stream()) == 0, lib.xunet_last_error()
    ref = torch.cat([x @ w.float().double() + b.float().double() for w, b in zip(ws, bs)], dim=-1)
    assert rel_l2(y.float(), ref) < TOL[dtype]
    dy = torch.randn(ref.shape, generator=g, dtype=torch.float64).to(DT[dtype]).double()
    dyd = dy.to(DT[dtype]).cuda()
    dx = torch.zeros(N, H, W, Cc, dtype=DT[dtype], device='cuda')
    assert lib.xunet_op_conv_dgrad(dtype, 0, dyd.data_ptr(), wflat.data_ptr(), dx.data_ptr(), N, H, W, Cc, 3 * Cc, 1, 1, 3,
                                   1.0, 0, _stream()) == 0
    dx_ref = sum(dy[..., i * Cc:(i + 1) * Cc] @ ws[i].float().double().T for i in range(3))
    assert rel_l2(dx.float(), dx_ref) < TOL[dtype]
    dw = torch.zeros(3 * Cc * Cc, dtype=torch.float32, device='cuda')
    db = torch.zeros(3 * Cc, dtype=torch.float32, device='cuda')
    assert lib.xunet_op_conv_wgrad(dtype, 0, xd.data_ptr(), dyd.data_ptr(), dw.data_ptr(), db.data_ptr(), N, H, W, Cc, 3 * Cc,
                                   1, 1, 3, 1.0, _stream()) == 0
    x2 = x.reshape(-1, Cc)
    dw_ref = torch.cat([(x2.T @ dy.reshape(-1, 3 * Cc)[:, i * Cc:(i + 1) * Cc]).reshape(-1) for i in range(3)])
    assert rel_l2(dw, dw_ref) < TOL[dtype]
    assert rel_l2(db, dy.reshape(-1, 3 * Cc).sum(0)) < TOL[dtype]


ATTN_CASES = [(2, 64, 32, 2, 0), (2, 64, 32, 2, 1), (4, 256, 64, 4, 1), (2, 1024, 64, 4, 0), (2, 64, 128, 2, 1),
              (2, 64, 128, 1, 0), (2, 48, 32, 2, 1)]


@pytest.mark.parametrize('dtype', [0, 1])
@pytest.mark.parametrize('case', ATTN_CASES)
def test_attention_fwd_bwd(lib, dtype, case):
    N, L, Cc, heads, cross = case
    hd = Cc // heads
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    qkv = (torch.randn(N, L, 3 * Cc, generator=g, dtype=torch.float64) * 1.5).to(DT[dtype]).double().requires_grad_(True)
    res = torch.randn(N, L, Cc, generator=g, dtype=torch.float64).to(DT[dtype]).double().requires_grad_(True)
    q, k, v = [t.reshape(N, L, heads, hd) for t in torch.split(qkv, Cc, dim=-1)]
    if cross:
        perm = torch.arange(N) ^ 1
        k, v = k[perm], v[perm]
    w = torch.softmax(torch.einsum('nqhd,nkhd->nhqk', q / math.sqrt(hd), k), dim=-1)
    o = torch.einsum('nhqk,nkhd->nqhd', w, v).reshape(N, L, Cc)
    out_ref = (o + res) / math.sqrt(2)
    dout = torch.randn(N, L, Cc, generator=g, dtype=torch.float64).to(DT[dtype]).double()
    out_ref.backward(dout)

    qd = qkv.detach().to(DT[dtype]).cuda().contiguous()
    rd = res.detach().to(DT[dtype]).cuda().contiguous()
    od = torch.zeros(N, L, Cc, dtype=DT[dtype], device='cuda')
    lse = torch.zeros(N, heads, L, dtype=torch.float32, device='cuda')
    assert lib.xunet_op_attention(dtype, 0, qd.data_ptr(), rd.data_ptr(), od.data_ptr(), lse.data_ptr(), N, L, Cc, heads,
                                  cross, _stream()) == 0, lib.xunet_last_error()
    assert rel_l2(od.float(), out_ref.detach()) < TOL[dtype]
    dd = dout.to(DT[dtype]).cuda().contiguous()
    scratch = torch.zeros(N * L * (heads + Cc), dtype=torch.float32, device='cuda')
    dqkv = torch.zeros(N, L, 3 * Cc, dtype=DT[dtype], device='cuda')
    # feed the exact forward output the kernel produced (it recomputes attn = out*sqrt2 - res from it)
    assert lib.xunet_op_attention_bwd(dtype, 0, qd.data_ptr(), rd.data_ptr(), od.data_ptr(), dd.data_ptr(), lse.data_ptr(),
                                      scratch.data_ptr(), dqkv.data_ptr(), N, L, Cc, heads, cross, _stream()) == 0
    assert rel_l2(dqkv.float(), qkv.grad) < (3e-5 if dtype == 0 else 4e-2)


def test_adam_matches_optax_formula(lib):
    g = torch.Generator().manual_seed(0)
    n = 10007
    p = torch.randn(n, generator=g, dtype=torch.float64)
    m = torch.zeros(n, dtype=torch.float64)
    v = torch.zeros(n, dtype=torch.float64)
    pd, md, vd = p.float().cuda(), m.float().cuda(), v.float().cuda()
    for step in range(1, 4):
        gr = torch.randn(n, generator=g, dtype=torch.float64)
        p, m, v = R.adam_update(p, gr * 0.5, m, v, step, lr=1e-3)
        gd = gr.float().cuda()
        assert lib.xunet_adam_step(pd.data_ptr(), gd.data_ptr(), md.data_ptr(), vd.data_ptr(), n, step, None, 1e-3, 0.9, 0.999,
                                   1e-8, 0.5, _stream()) == 0
    assert rel_l2(pd, p) < 1e-6 and rel_l2(md, m) < 1e-6 and rel_l2(vd, v) < 1e-6
    # first step from zero moments moves by -lr*sign(g)  (SURVEY 8c item 9)
    p0 = torch.zeros(16, device='cuda'); m0 = torch.zeros(16, device='cuda'); v0 = torch.zeros(16, device='cuda')
    g0 = torch.linspace(-1, 1, 16, device='cuda') + 0.03
    lib.xunet_adam_step(p0.data_ptr(), g0.data_ptr(), m0.data_ptr(), v0.data_ptr(), 16, 1, None, 1e-4, 0.9, 0.999, 1e-8, 1.0, _stream())
    assert torch.allclose(p0, -1e-4 * torch.sign(g0), atol=1e-9)


def test_dropout_mask_matches_numpy_replica(lib):
    from tests.util import keep_mask
    n = 64 * 64 * 32
    out = torch.zeros(n, device='cuda')
    assert lib.xunet_dropout_mask(out.data_ptr(), n, 5, 123456789, 0.1, _stream()) == 0
    assert np.array_equal(out.cpu().numpy() > 0.5, keep_mask(123456789, 5, (n,), 0.1))


def test_sampler_step_table_matches_oracle(lib):
    """Loop positions k = 0..3 on table rows t = 999, 500, 1, 0, with explicit noise laid out (steps, n): step k must use row
    k and noise row k, and hand its z and row k's log-SNR to the next forward."""
    g = torch.Generator().manual_seed(4)
    tab = R.schedule_tables()
    ts = (999, 500, 1, 0)
    n, b2 = 2 * 8 * 8 * 3, 4
    rows = [[tab['sqrt_recip_alphas_cumprod'][t], tab['sqrt_recipm1_alphas_cumprod'][t], tab['posterior_mean_coef1'][t],
             tab['posterior_mean_coef2'][t], 0.0 if t == 0 else math.exp(0.5 * tab['posterior_log_variance_clipped'][t]),
             R.logsnr_schedule_cosine(t / 1000.0), 0.0, 0.0] for t in ts]
    tabd = torch.tensor(rows, dtype=torch.float64).float().cuda()
    noise = torch.randn(len(ts), n, generator=g, dtype=torch.float64)
    nd = noise.float().cuda()
    pos = torch.zeros(1, dtype=torch.int32, device='cuda')
    seed = torch.zeros(1, dtype=torch.int64, device='cuda')
    next_z2, next_logsnr2 = torch.zeros(2 * n, device='cuda'), torch.zeros(b2, device='cuda')
    for k, t in enumerate(ts):
        ec, eu, z = [torch.randn(n, generator=g, dtype=torch.float64) for _ in range(3)]
        ref, _ = R.sampler_step(ec, eu, z, t, noise[k], tab)
        eps2 = torch.cat([ec, eu]).float().cuda()
        zd = z.float().cuda()
        assert lib.xunet_sampler_step_table(eps2.data_ptr(), zd.data_ptr(), nd.data_ptr(), n, 3.0, tabd.data_ptr(), pos.data_ptr(),
                                            seed.data_ptr(), next_z2.data_ptr(), next_logsnr2.data_ptr(), b2, _stream()) == 0, \
            lib.xunet_last_error()
        pos.add_(1)
        # at t=999 sqrt(1/abar) ~ 6e4 amplifies fp32 rounding before the clip; compare on the clipped scale
        assert float((zd.double().cpu() - ref).abs().max()) < 5e-3 if t == 999 else rel_l2(zd, ref) < 1e-5
        assert torch.equal(next_z2[:n], zd) and torch.equal(next_z2[n:], zd)
        assert bool((next_logsnr2 == tabd[k, 5]).all())
    # device-side noise (noise == NULL): unit variance, zero mean
    big = 1 << 20
    eps2 = torch.zeros(2 * big, device='cuda'); zz = torch.zeros(big, device='cuda'); zz2 = torch.zeros(2 * big, device='cuda')
    unit = torch.tensor([[1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]], device='cuda')      # z' = 1 * noise
    pos.zero_(); seed.fill_(77)
    assert lib.xunet_sampler_step_table(eps2.data_ptr(), zz.data_ptr(), None, big, 3.0, unit.data_ptr(), pos.data_ptr(),
                                        seed.data_ptr(), zz2.data_ptr(), next_logsnr2.data_ptr(), b2, _stream()) == 0
    assert abs(float(zz.mean())) < 5e-3 and abs(float(zz.std()) - 1.0) < 5e-3


# ----------------------------------------------------------------------------------------------------------------
# wgmma / TMA implicit-GEMM convolution (impl=1) against the fp64 restatement (and therefore the SIMT kernel)
# ----------------------------------------------------------------------------------------------------------------
TC_CASES = [
    # N, H, W, Ci, Co, ks, nseg
    (16, 64, 64, 32, 32, 3, 1), (16, 32, 32, 64, 64, 3, 1), (16, 32, 32, 128, 64, 3, 1), (16, 32, 32, 96, 64, 3, 1),
    (4, 64, 64, 96, 32, 3, 1), (16, 32, 32, 64, 192, 1, 3), (16, 32, 32, 32, 128, 1, 1), (16, 64, 64, 64, 32, 1, 1),
    (4, 16, 16, 64, 64, 3, 1), (4, 8, 8, 64, 64, 3, 1), (2, 128, 128, 32, 32, 3, 1), (2, 32, 32, 256, 512, 3, 1),
    (2, 64, 64, 144, 32, 3, 1),
]


@pytest.mark.parametrize('case', TC_CASES)
def test_conv_tcgen05_fwd_and_dgrad(lib, case):
    N, H, W, Ci, Co, ks, nseg = case
    dtype = 1
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    taps = ks * ks
    x = torch.randn(N, H, W, Ci, generator=g, dtype=torch.float32).to(torch.bfloat16)
    segw = Co // nseg
    w = (torch.randn(nseg, taps, Ci, segw, generator=g, dtype=torch.float32) / math.sqrt(taps * Ci))
    b = torch.randn(Co, generator=g, dtype=torch.float32) * 0.1
    wq = w.to(torch.bfloat16).double()                       # the kernel multiplies bf16-rounded weights
    wfull = torch.cat([wq[sgi] for sgi in range(nseg)], dim=-1)   # (taps, Ci, Co)
    xr = x.double().requires_grad_(True)
    y_ref = _ref_conv(xr, wfull, b.double(), 1, ks)
    res = torch.randn(y_ref.shape, generator=g, dtype=torch.float32).to(torch.bfloat16)
    alpha = 0.7071
    out_ref = (y_ref + res.double()) * alpha
    dy = torch.randn(y_ref.shape, generator=g, dtype=torch.float32).to(torch.bfloat16)
    out_ref.backward(dy.double())

    xd, wd, bd, rd = x.cuda(), w.cuda().contiguous(), b.cuda(), res.cuda()
    yd = torch.zeros(N, H, W, Co, dtype=torch.bfloat16, device='cuda')
    rc = lib.xunet_op_conv(dtype, 1, xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), rd.data_ptr(), yd.data_ptr(), N, H, W, Ci, Co,
                           ks, 1, nseg, alpha, _stream())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    assert rel_l2(yd.float(), out_ref.detach()) < 6e-3      # only the bf16 rounding of the output remains

    if Ci % 32 == 0:
        dyd = dy.cuda()
        dxd = torch.zeros(N, H, W, Ci, dtype=torch.bfloat16, device='cuda')
        rc = lib.xunet_op_conv_dgrad(dtype, 1, dyd.data_ptr(), wd.data_ptr(), dxd.data_ptr(), N, H, W, Ci, Co, ks, 1, nseg,
                                     alpha, 0, _stream())
        assert rc == 0, lib.xunet_last_error()
        torch.cuda.synchronize()
        assert rel_l2(dxd.float(), xr.grad) < 6e-3
        rc = lib.xunet_op_conv_dgrad(dtype, 1, dyd.data_ptr(), wd.data_ptr(), dxd.data_ptr(), N, H, W, Ci, Co, ks, 1, nseg,
                                     alpha, 1, _stream())
        assert rc == 0
        torch.cuda.synchronize()
        assert rel_l2(dxd.float(), 2 * xr.grad) < 1e-2

    # weight / bias gradient on the tensor cores (exact bf16 products, fp32 accumulation -> tight tolerance)
    wr = wfull.clone().requires_grad_(True)
    br = b.double().requires_grad_(True)
    ((_ref_conv(x.double(), wr, br, 1, ks)) * alpha).backward(dy.double())
    dw_ref = torch.stack([wr.grad[..., sgi * segw:(sgi + 1) * segw] for sgi in range(nseg)])     # (nseg, taps, Ci, segw)
    dwd = torch.zeros(nseg, taps, Ci, segw, dtype=torch.float32, device='cuda')
    dbd = torch.zeros(Co, dtype=torch.float32, device='cuda')
    rc = lib.xunet_op_conv_wgrad(dtype, 1, xd.data_ptr(), dy.cuda().data_ptr(), dwd.data_ptr(), dbd.data_ptr(), N, H, W, Ci, Co,
                                 ks, 1, nseg, alpha, _stream())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    assert rel_l2(dwd, dw_ref) < 1e-4
    assert rel_l2(dbd, br.grad) < 1e-4


ATTN_TC_CASES = [(2, 128, 32, 2, 0), (2, 256, 64, 4, 1), (4, 1024, 64, 4, 0), (4, 1024, 64, 4, 1), (2, 256, 64, 2, 0),
                 (2, 256, 128, 2, 1), (2, 256, 128, 1, 0), (2, 256, 256, 2, 1)]


@pytest.mark.parametrize('case', ATTN_TC_CASES)
def test_attention_tcgen05_fwd(lib, case):
    N, L, Cc, heads, cross = case
    hd = Cc // heads
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    qkv = (torch.randn(N, L, 3 * Cc, generator=g, dtype=torch.float32) * 1.5).to(torch.bfloat16)
    res = torch.randn(N, L, Cc, generator=g, dtype=torch.float32).to(torch.bfloat16)
    q, k, v = [t.double().reshape(N, L, heads, hd) for t in torch.split(qkv, Cc, dim=-1)]
    if cross:
        perm = torch.arange(N) ^ 1
        k, v = k[perm], v[perm]
    sc = torch.einsum('nqhd,nkhd->nhqk', q / math.sqrt(hd), k)
    w = torch.softmax(sc, dim=-1)
    o = torch.einsum('nhqk,nkhd->nqhd', w, v).reshape(N, L, Cc)
    out_ref = (o + res.double()) / math.sqrt(2)
    lse_ref = torch.logsumexp(sc, dim=-1)
    qd, rd = qkv.cuda(), res.cuda()
    od = torch.zeros(N, L, Cc, dtype=torch.bfloat16, device='cuda')
    lse = torch.zeros(N, heads, L, dtype=torch.float32, device='cuda')
    rc = lib.xunet_op_attention(1, 1, qd.data_ptr(), rd.data_ptr(), od.data_ptr(), lse.data_ptr(), N, L, Cc, heads, cross, _stream())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    assert rel_l2(lse, lse_ref) < 1e-4
    assert rel_l2(od.float(), out_ref) < 8e-3          # P is rounded to bf16 before the PV tensor-core GEMM


@pytest.mark.parametrize('case', ATTN_TC_CASES)
def test_attention_tcgen05_bwd(lib, case):
    N, L, Cc, heads, cross = case
    hd = Cc // heads
    g = torch.Generator().manual_seed(hash(case) & 0xFFF)
    qkv = (torch.randn(N, L, 3 * Cc, generator=g, dtype=torch.float32) * 1.5).to(torch.bfloat16)
    res = torch.randn(N, L, Cc, generator=g, dtype=torch.float32).to(torch.bfloat16)
    dout = torch.randn(N, L, Cc, generator=g, dtype=torch.float32).to(torch.bfloat16)
    qr = qkv.double().requires_grad_(True)
    q, k, v = [t.reshape(N, L, heads, hd) for t in torch.split(qr, Cc, dim=-1)]
    if cross:
        perm = torch.arange(N) ^ 1
        k, v = k[perm], v[perm]
    w = torch.softmax(torch.einsum('nqhd,nkhd->nhqk', q / math.sqrt(hd), k), dim=-1)
    o = torch.einsum('nhqk,nkhd->nqhd', w, v).reshape(N, L, Cc)
    ((o + res.double()) / math.sqrt(2)).backward(dout.double())
    qd, rd, dd = qkv.cuda(), res.cuda(), dout.cuda()
    od = torch.zeros(N, L, Cc, dtype=torch.bfloat16, device='cuda')
    lse = torch.zeros(N, heads, L, dtype=torch.float32, device='cuda')
    assert lib.xunet_op_attention(1, 1, qd.data_ptr(), rd.data_ptr(), od.data_ptr(), lse.data_ptr(), N, L, Cc, heads, cross, _stream()) == 0
    scratch = torch.zeros(N * L * (heads + Cc), dtype=torch.float32, device='cuda')
    dqkv = torch.zeros(N, L, 3 * Cc, dtype=torch.bfloat16, device='cuda')
    rc = lib.xunet_op_attention_bwd(1, 1, qd.data_ptr(), rd.data_ptr(), od.data_ptr(), dd.data_ptr(), lse.data_ptr(),
                                    scratch.data_ptr(), dqkv.data_ptr(), N, L, Cc, heads, cross, _stream())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    gq, gk, gv = [rel_l2(a.float(), b) for a, b in zip(torch.split(dqkv, Cc, dim=-1), torch.split(qr.grad, Cc, dim=-1))]
    assert max(gq, gk, gv) < 4e-2, (gq, gk, gv)


@pytest.mark.parametrize('dtype', [0, 1])
@pytest.mark.parametrize('case', [(4, 16, 16, 3, 32), (2, 32, 32, 3, 64), (4, 16, 16, 32, 3), (2, 32, 32, 64, 3),
                                  (2, 64, 64, 3, 256), (2, 64, 64, 256, 3),      # the 3DiM widths: 32 lanes per pixel quad
                                  (2, 8, 48, 3, 32), (2, 8, 48, 32, 3),          # W % 32 != 0: round-1 wgrad kernels, new fwd / dgrad
                                  (2, 12, 20, 3, 32), (2, 12, 20, 32, 3),        # W < 32: one segment per row
                                  (2, 6, 6, 3, 16), (2, 6, 6, 16, 3),            # W % 4 != 0: round-1 kernels throughout
                                  (2, 8, 8, 3, 896)])                            # the input conv at ch = 896: > 96 KiB of weights in smem
def test_three_channel_direct_convs(lib, dtype, case):
    """impl=2: the direct kernels for the input conv (Cin=3) and the output conv (Cout=3)."""
    N, H, W, Ci, Co = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    x = torch.randn(N, H, W, Ci, generator=g, dtype=torch.float64).to(DT[dtype]).double()
    w = (torch.randn(9, Ci, Co, generator=g, dtype=torch.float64) / math.sqrt(9 * Ci)).float().double()
    b = (torch.randn(Co, generator=g, dtype=torch.float64) * 0.1).float().double()
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y_ref = _ref_conv(xr, wr, br, 1, 3)
    dy = torch.randn(y_ref.shape, generator=g, dtype=torch.float64).to(DT[dtype]).double()
    y_ref.backward(dy)
    xd, wd, bd = x.to(DT[dtype]).cuda(), w.float().cuda(), b.float().cuda()
    yd = torch.zeros(N, H, W, Co, dtype=DT[dtype], device='cuda')
    assert lib.xunet_op_conv(dtype, 2, xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), None, yd.data_ptr(), N, H, W, Ci, Co, 3, 1, 1,
                             1.0, _stream()) == 0, lib.xunet_last_error()
    assert rel_l2(yd.float(), y_ref.detach()) < TOL[dtype]
    dyd = dy.to(DT[dtype]).cuda()
    dw = torch.zeros(9, Ci, Co, dtype=torch.float32, device='cuda')
    db = torch.zeros(Co, dtype=torch.float32, device='cuda')
    assert lib.xunet_op_conv_wgrad(dtype, 2, xd.data_ptr(), dyd.data_ptr(), dw.data_ptr(), db.data_ptr(), N, H, W, Ci, Co, 3, 1, 1,
                                   1.0, _stream()) == 0, lib.xunet_last_error()
    assert rel_l2(dw, wr.grad) < TOL[dtype] and rel_l2(db, br.grad) < TOL[dtype]
    if Co == 3:
        dx = torch.zeros(N, H, W, Ci, dtype=DT[dtype], device='cuda')
        assert lib.xunet_op_conv_dgrad(dtype, 2, dyd.data_ptr(), wd.data_ptr(), dx.data_ptr(), N, H, W, Ci, Co, 3, 1, 1, 1.0, 0,
                                       _stream()) == 0, lib.xunet_last_error()
        assert rel_l2(dx.float(), xr.grad) < TOL[dtype]
        assert lib.xunet_op_conv_dgrad(dtype, 2, dyd.data_ptr(), wd.data_ptr(), dx.data_ptr(), N, H, W, Ci, Co, 3, 1, 1, 1.0, 1,
                                       _stream()) == 0
        assert rel_l2(dx.float(), 2 * xr.grad) < 2 * TOL[dtype]


@pytest.mark.parametrize('case', [(4, 64, 64, 144, 32, 2), (2, 128, 128, 144, 64, 4), (2, 128, 128, 144, 64, 8), (4, 32, 32, 64, 64, 2)])
def test_conv_tcgen05_strided_forward_and_wgrad(lib, case):
    """The pose-embedding convs (model/xunet.py:197-202): 3x3, stride 2^level, SAME -> TMA traversal strides."""
    N, H, W, Ci, Co, stride = case
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    x = torch.randn(N, H, W, Ci, generator=g, dtype=torch.float32).to(torch.bfloat16)
    w = torch.randn(9, Ci, Co, generator=g, dtype=torch.float32) / math.sqrt(9 * Ci)
    b = torch.randn(Co, generator=g, dtype=torch.float32) * 0.1
    wq = w.to(torch.bfloat16).double().requires_grad_(True)
    br = b.double().requires_grad_(True)
    y_ref = _ref_conv(x.double(), wq, br, stride, 3)
    Ho, Wo = y_ref.shape[1], y_ref.shape[2]
    dy = torch.randn(y_ref.shape, generator=g, dtype=torch.float32).to(torch.bfloat16)
    y_ref.backward(dy.double())
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    yd = torch.zeros(N, Ho, Wo, Co, dtype=torch.bfloat16, device='cuda')
    assert lib.xunet_op_conv(1, 1, xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), None, yd.data_ptr(), N, H, W, Ci, Co, 3, stride, 1,
                             1.0, _stream()) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    assert rel_l2(yd.float(), y_ref.detach()) < 6e-3
    dw = torch.zeros(9, Ci, Co, dtype=torch.float32, device='cuda')
    db = torch.zeros(Co, dtype=torch.float32, device='cuda')
    assert lib.xunet_op_conv_wgrad(1, 1, xd.data_ptr(), dy.cuda().data_ptr(), dw.data_ptr(), db.data_ptr(), N, H, W, Ci, Co, 3,
                                   stride, 1, 1.0, _stream()) == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    assert rel_l2(dw, wq.grad) < 1e-4 and rel_l2(db, br.grad) < 1e-4


@pytest.mark.parametrize('case', [(2, 128, 32, 2, 0), (4, 1024, 64, 4, 1), (2, 256, 64, 2, 0), (2, 256, 64, 4, 1)])
def test_attention_tcgen05_bwd_single_kernel_fold(lib, case, monkeypatch):
    """XUNET_OP_ATTN_FOLD=1: the caller keeps its scratch buffer all-zero between calls and the backward (prep, dK/dV/dQ,
    dQ store) hands it back all-zero (the store kernel re-zeroes the D rows): correct gradients, scratch all-zero afterwards,
    and a second call on the same scratch gives the same gradients."""
    monkeypatch.setenv('XUNET_OP_ATTN_FOLD', '1')
    N, L, Cc, heads, cross = case
    hd = Cc // heads
    assert hd <= 32
    g = torch.Generator().manual_seed(hash(case) & 0xFFF)
    qkv = (torch.randn(N, L, 3 * Cc, generator=g, dtype=torch.float32) * 1.5).to(torch.bfloat16)
    res = torch.randn(N, L, Cc, generator=g, dtype=torch.float32).to(torch.bfloat16)
    dout = torch.randn(N, L, Cc, generator=g, dtype=torch.float32).to(torch.bfloat16)
    qr = qkv.double().requires_grad_(True)
    q, k, v = [t.reshape(N, L, heads, hd) for t in torch.split(qr, Cc, dim=-1)]
    if cross:
        perm = torch.arange(N) ^ 1
        k, v = k[perm], v[perm]
    w = torch.softmax(torch.einsum('nqhd,nkhd->nhqk', q / math.sqrt(hd), k), dim=-1)
    o = torch.einsum('nhqk,nkhd->nqhd', w, v).reshape(N, L, Cc)
    ((o + res.double()) / math.sqrt(2)).backward(dout.double())
    qd, rd, dd = qkv.cuda(), res.cuda(), dout.cuda()
    od = torch.zeros(N, L, Cc, dtype=torch.bfloat16, device='cuda')
    lse = torch.zeros(N, heads, L, dtype=torch.float32, device='cuda')
    assert lib.xunet_op_attention(1, 1, qd.data_ptr(), rd.data_ptr(), od.data_ptr(), lse.data_ptr(), N, L, Cc, heads, cross, _stream()) == 0
    scratch = torch.zeros(N * L * (heads + Cc), dtype=torch.float32, device='cuda')
    outs = []
    for _ in range(2):
        dqkv = torch.full((N, L, 3 * Cc), float('nan'), dtype=torch.bfloat16, device='cuda')
        rc = lib.xunet_op_attention_bwd(1, 1, qd.data_ptr(), rd.data_ptr(), od.data_ptr(), dd.data_ptr(), lse.data_ptr(),
                                        scratch.data_ptr(), dqkv.data_ptr(), N, L, Cc, heads, cross, _stream())
        assert rc == 0, lib.xunet_last_error()
        torch.cuda.synchronize()
        assert float(scratch.abs().max()) == 0.0                      # D rows left clean
        gq, gk, gv = [rel_l2(a.float(), b) for a, b in zip(torch.split(dqkv, Cc, dim=-1), torch.split(qr.grad, Cc, dim=-1))]
        assert max(gq, gk, gv) < 4e-2, (gq, gk, gv)
        outs.append(dqkv.float().clone())
    assert rel_l2(outs[1], outs[0]) < 1e-3                            # same inputs, same gradients
