"""Every conv and attention launch of the plans bench.py measures, element by element against fp64 (tests/launch_ref.py).

The launch list comes from the plans themselves (xunet_plan_launch), deduplicated by everything that changes a launch, and
each launch runs through the operator-level entry point with the plan's kernel (impl), at the plan's exact shape:
  * conv: the forward (xunet_op_conv, or xunet_op_conv_stats where the plan's epilogue emits the GroupNorm statistics), the
    data gradient (xunet_op_conv_dgrad with the plan's alpha and accumulate flag, or xunet_op_conv_dgrad_groupnorm where the
    plan fuses the GroupNorm backward into it) and the weight gradient (xunet_op_conv_wgrad);
  * attention: the forward (with statistics where the plan emits them) and, in training plans, the backward, each on a
    moderate input and on a peaked one whose largest scores lie in the last 64-key block.
Inputs carry per-frame and per-channel offsets, so that a routing error between samples, frames, heads or channels shows.  Each
check prints the worst err / bound and the element where it occurs.  The fp64 references run on the GPU."""
import math
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

from novel_view_synthesis_3d_b200 import _lib
from tests import groupnorm_ref as G
from tests import launch_ref as L
from tests.test_gpu_groupnorm import _check_epi, _run_epi

pytestmark = pytest.mark.gpu

F64 = torch.float64
DT = {0: torch.float32, 1: torch.bfloat16}
IMPL = {_lib.KERNEL_SIMT: 0, _lib.KERNEL_TC: 1, _lib.KERNEL_CIN3: 2, _lib.KERNEL_COUT3: 2}
UNIQUE = L.unique_launches(_lib.load())
CONVS = [u for u in UNIQUE if u[3]['kind'] == _lib.LAUNCH_CONV]
ATTNS = [u for u in UNIQUE if u[3]['kind'] == _lib.LAUNCH_ATTN]


def _s():
    return torch.cuda.current_stream().cuda_stream


def _gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def _rand(shape, g, scale=1.):
    return (torch.randn(shape, generator=g, dtype=F64) * scale).cuda()


def _q(t, dtype):
    """round to the storage type and back to fp64: the kernel's input"""
    return t.to(DT[dtype]).to(F64)


def _offsets(N, C):
    """per-frame and per-channel offsets of an (N, ..., C) input"""
    return (0.3 * torch.arange(N, dtype=F64)[:, None, None, None] + 0.1 * torch.cos(torch.arange(C, dtype=F64))).cuda()


def _check(name, what, got, ref, bound):
    ratio, i, nbad = L.excess(got, ref, bound)
    idx = tuple(int(v) for v in np.unravel_index(i, tuple(ref.shape)))
    print(f'{name} {what}: worst err/bound {ratio:.3g} at {idx}')
    assert nbad == 0, (f'{name} {what}: {nbad} of {ref.numel()} elements out of bounds; worst at {idx}: got '
                       f'{float(got.reshape(-1)[i]):.6g}, ref {float(ref.reshape(-1)[i]):.6g}, bound {float(bound.reshape(-1)[i]):.3g}')


def check_conv(lib, case, plans=L.PLANS):
    """the forward, data gradient and weight gradient of one conv launch (name, dtype, training, launch) of `plans` against fp64"""
    name, dtype, training, r = case
    N, Hi, Wi, Ci, Ho, Wo, Co = (r[k] for k in ('N', 'Hi', 'Wi', 'Ci', 'Ho', 'Wo', 'Co'))
    ks, st, nseg, alpha, balpha = r['ksize'], r['stride'], r['nseg'], r['alpha'], r['bwd_alpha']
    bf = dtype == 1
    taps = ks * ks
    g = _gen(name)
    x = _q(_rand((N, Hi, Wi, Ci), g) + _offsets(N, Ci), dtype)
    w = _rand((taps * Ci * Co,), g, 1 / math.sqrt(taps * Ci)).float()
    b = _rand((Co,), g, 0.3).float()
    res = _q(_rand((N, Ho, Wo, Co), g) + _offsets(N, Co), dtype) if r['residual'] else None
    # the weights each kernel multiplies: the bf16 shadow on the tensor cores, the fp32 master weights elsewhere
    wk = {k: L.weight((w.to(torch.bfloat16) if k == _lib.KERNEL_TC else w).to(F64), ks, Ci, Co, nseg) for k in IMPL}
    xd = x.to(DT[dtype])
    rd = res.to(DT[dtype]) if res is not None else None
    y = torch.zeros(N, Ho, Wo, Co, dtype=DT[dtype], device='cuda')
    if r['emits_stats']:
        cs = torch.zeros(N // 2, Co, 2, dtype=torch.float32, device='cuda')
        rc = lib.xunet_op_conv_stats(dtype, IMPL[r['fwd']], xd.data_ptr(), w.data_ptr(), b.data_ptr(),
                                     rd.data_ptr() if rd is not None else None, y.data_ptr(), cs.data_ptr(), N, Hi, Wi, Ci, Co, ks,
                                     alpha, _s())
    else:
        rc = lib.xunet_op_conv(dtype, IMPL[r['fwd']], xd.data_ptr(), w.data_ptr(), b.data_ptr(),
                               rd.data_ptr() if rd is not None else None, y.data_ptr(), N, Hi, Wi, Ci, Co, ks, st, nseg, alpha, _s())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    ref, bound = L.conv_fwd_check(x, wk[r['fwd']], b.to(F64), res, alpha, ks, st, bf)
    _check(name, 'forward', y, ref, bound)
    del ref, bound
    if r['emits_stats']:
        # the epilogue's [sum, sumsq] of the stored output: fp32 over 32-row slices, fp64 across them (tests/test_gpu_groupnorm.py)
        y64 = y.to(F64)
        _check(name, 'forward cstats', cs, G.cstats(y64), 1e-6 * G.cstats(y64.abs()) + 1e-30)
        del y64
    if r['dgrad'] == _lib.KERNEL_NONE and r['wgrad'] == _lib.KERNEL_NONE:
        return
    dy = _q(_rand((N, Ho, Wo, Co), g) + _offsets(N, Co), dtype)
    dyd = dy.to(DT[dtype])
    if r['gn_mode'] >= 0:
        # the data gradient carries the GroupNorm backward: the fused epilogue at this shape and mode
        cfg_rate = L.plan_config(plans[name.split(':')[0]][0]).dropout
        rg = torch.Generator().manual_seed(zlib.crc32((name + ':epi').encode()))
        ep = _run_epi(lib, rg, N, Hi, Wi, Ci, Co, ks, nseg, r['gn_mode'], balpha, cfg_rate, 1)
        _check_epi(ep, N, Hi, Wi, Ci, Co, ks, nseg, r['gn_mode'], balpha, cfg_rate, 1)
        print(f'{name} dgrad + GroupNorm backward (mode {r["gn_mode"]}): within bounds')
        del ep
    elif r['dgrad'] != _lib.KERNEL_NONE:
        # the destination holds a non-zero prior: added to when the launch accumulates, overwritten otherwise
        prior = _q(_rand((N, Hi, Wi, Ci), g) + _offsets(N, Ci), dtype)
        dx = prior.to(DT[dtype])
        rc = lib.xunet_op_conv_dgrad(dtype, IMPL[r['dgrad']], dyd.data_ptr(), w.data_ptr(), dx.data_ptr(), N, Hi, Wi, Ci, Co, ks, st,
                                     nseg, balpha, r['accumulate'], _s())
        assert rc == 0, lib.xunet_last_error()
        torch.cuda.synchronize()
        ref, bound = L.conv_dgrad_check(dy, wk[r['dgrad']], balpha, ks, st, Hi, Wi, bf, prior if r['accumulate'] else None)
        _check(name, f'dgrad (accumulate={r["accumulate"]})', dx, ref, bound)
        del ref, bound, dx, prior
    if r['wgrad'] != _lib.KERNEL_NONE:
        dw0 = _rand((taps * Ci * Co,), g, 0.01).float()
        db0 = _rand((Co,), g, 0.01).float()
        dw, db = dw0.clone(), db0.clone()
        rc = lib.xunet_op_conv_wgrad(dtype, IMPL[r['wgrad']], xd.data_ptr(), dyd.data_ptr(), dw.data_ptr(), db.data_ptr(), N, Hi, Wi,
                                     Ci, Co, ks, st, nseg, balpha, _s())
        assert rc == 0, lib.xunet_last_error()
        torch.cuda.synchronize()
        rdw, bdw, rdb, bdb = L.conv_wgrad_check(x, dy, balpha, ks, st, L.weight(dw0.to(F64), ks, Ci, Co, nseg), db0.to(F64))
        _check(name, 'wgrad dW', dw, L.weight_flat(rdw, nseg), L.weight_flat(bdw, nseg))
        _check(name, 'wgrad dbias', db, rdb, bdb)


def check_attention(lib, case, peaked):
    """the forward and, in a training plan, the backward of one attention launch (name, dtype, training, launch) against fp64"""
    name, dtype, training, r = case
    N, Lk, C, heads, cross, impl = (r[k] for k in ('N', 'L', 'C', 'heads', 'cross', 'impl'))
    bf = dtype == 1
    g = _gen(name + str(peaked))
    qkv = _q(L.attn_qkv(N, Lk, C, heads, peaked, g).cuda(), dtype)
    res = _q(_rand((N, Lk, 1, C), g) + _offsets(N, C), dtype).reshape(N, Lk, C)
    qd, rd = qkv.to(DT[dtype]), res.to(DT[dtype])
    out = torch.zeros(N, Lk, C, dtype=DT[dtype], device='cuda')
    lse = torch.zeros(N, heads, Lk, dtype=torch.float32, device='cuda')
    if r['emits_stats']:
        cs = torch.zeros(N // 2, C, 2, dtype=torch.float32, device='cuda')
        rc = lib.xunet_op_attention_stats(dtype, impl, qd.data_ptr(), rd.data_ptr(), out.data_ptr(), lse.data_ptr(), cs.data_ptr(),
                                          N, Lk, C, heads, cross, _s())
    else:
        rc = lib.xunet_op_attention(dtype, impl, qd.data_ptr(), rd.data_ptr(), out.data_ptr(), lse.data_ptr(), N, Lk, C, heads,
                                    cross, _s())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    ref, bound, lref, lbound = L.attn_fwd_check(qkv, res, heads, cross, bf)
    _check(name, 'attention out', out, ref, bound)
    _check(name, 'attention lse', lse, lref, lbound)
    # chain: the exact fp64 forward of the bf16 inputs at the operator tests' rel-L2 tolerance
    rel = float(torch.linalg.norm(out.to(F64) - ref) / torch.linalg.norm(ref))
    assert rel < (8e-3 if bf else 1e-5), rel
    del ref, bound, lref, lbound
    if r['emits_stats']:
        o64 = out.to(F64).reshape(N, Lk, 1, C)
        _check(name, 'attention cstats', cs, G.cstats(o64), 1e-6 * G.cstats(o64.abs()) + 1e-30)
    if not training:
        return
    dout = _q(_rand((N, Lk, 1, C), g) + _offsets(N, C), dtype).reshape(N, Lk, C)
    dd = dout.to(DT[dtype])
    dscr = torch.zeros(N * heads * Lk, dtype=torch.float32, device='cuda')
    dqkv = _rand((N, Lk, 3 * C), g).to(DT[dtype])       # overwritten
    rc = lib.xunet_op_attention_bwd(dtype, impl, qd.data_ptr(), rd.data_ptr(), out.data_ptr(), dd.data_ptr(), lse.data_ptr(),
                                    dscr.data_ptr(), dqkv.data_ptr(), N, Lk, C, heads, cross, _s())
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()
    # stage: on the kernel's own inputs (its stored out and lse)
    ref, bound = L.attn_bwd_check(qkv, res, out.to(F64), dout, lse.to(F64), heads, cross, bf)
    _check(name, 'attention dqkv', dqkv, ref, bound)
    del ref, bound
    # chain: the exact fp64 backward of the bf16 inputs at the operator tests' rel-L2 tolerance
    ex = L.attn_bwd_exact(qkv, res, dout, heads, cross)
    rel = float(torch.linalg.norm(dqkv.to(F64) - ex) / torch.linalg.norm(ex))
    assert rel < (4e-2 if bf else 1e-4), rel


@pytest.mark.parametrize('case', CONVS, ids=[u[0] for u in CONVS])
def test_conv_launch(lib, case):
    check_conv(lib, case)


@pytest.mark.parametrize('peaked', [False, True], ids=['moderate', 'peaked'])
@pytest.mark.parametrize('case', ATTNS, ids=[u[0] for u in ATTNS])
def test_attention_launch(lib, case, peaked):
    check_attention(lib, case, peaked)


# ======================================================================================================================
# which tensor-core variants the plan-derived launches reach, read from the launchers' log in a child process
# ======================================================================================================================
def _launch_all_convs(cases=None):
    """every launch test_conv_launch checks (or those of `cases`), once more on zero-filled buffers and unchecked: what the
    variants tests log"""
    lib = _lib.load()
    for name, dtype, training, r in (CONVS if cases is None else cases):
        N, Hi, Wi, Ci, Ho, Wo, Co = (r[k] for k in ('N', 'Hi', 'Wi', 'Ci', 'Ho', 'Wo', 'Co'))
        ks, st, nseg = r['ksize'], r['stride'], r['nseg']
        z = lambda *shape, dt=DT[dtype]: torch.zeros(*shape, dtype=dt, device='cuda')
        x, y, dy, dx = z(N, Hi, Wi, Ci), z(N, Ho, Wo, Co), z(N, Ho, Wo, Co), z(N, Hi, Wi, Ci)
        w, b = z(ks * ks * Ci * Co, dt=torch.float32), z(Co, dt=torch.float32)
        res = z(N, Ho, Wo, Co) if r['residual'] else None
        cs = z(N // 2, Co, 2, dt=torch.float32)
        p = lambda t: None if t is None else t.data_ptr()
        if r['emits_stats']:
            rc = lib.xunet_op_conv_stats(dtype, IMPL[r['fwd']], p(x), p(w), p(b), p(res), p(y), p(cs), N, Hi, Wi, Ci, Co, ks,
                                         r['alpha'], _s())
        else:
            rc = lib.xunet_op_conv(dtype, IMPL[r['fwd']], p(x), p(w), p(b), p(res), p(y), N, Hi, Wi, Ci, Co, ks, st, nseg, r['alpha'],
                                   _s())
        assert rc == 0, lib.xunet_last_error()
        if r['gn_mode'] >= 0:
            film = r['gn_mode'] == G.FILM
            e, de = (z(N, Hi, Wi, 2 * Ci), z(N, Hi, Wi, 2 * Ci)) if film else (None, None)
            gp, bcs = z(N // 2, Ci, 4, dt=torch.float32), z(N // 2, Ci, 2, dt=torch.float32)
            rc = lib.xunet_op_conv_dgrad_groupnorm(dtype, p(dy), p(w), p(x), p(gp), r['gn_mode'], p(e), p(de), 0., 0, None, 0, p(dx),
                                                   p(bcs), N, Hi, Wi, Ci, Co, ks, nseg, r['bwd_alpha'], _s())
            assert rc == 0, lib.xunet_last_error()
        elif r['dgrad'] != _lib.KERNEL_NONE:
            rc = lib.xunet_op_conv_dgrad(dtype, IMPL[r['dgrad']], p(dy), p(w), p(dx), N, Hi, Wi, Ci, Co, ks, st, nseg, r['bwd_alpha'],
                                         r['accumulate'], _s())
            assert rc == 0, lib.xunet_last_error()
        if r['wgrad'] != _lib.KERNEL_NONE:
            dw = z(ks * ks * Ci * Co, dt=torch.float32)
            rc = lib.xunet_op_conv_wgrad(dtype, IMPL[r['wgrad']], p(x), p(dy), p(dw), p(b), N, Hi, Wi, Ci, Co, ks, st, nseg,
                                         r['bwd_alpha'], _s())
            assert rc == 0, lib.xunet_last_error()
        torch.cuda.synchronize()


def logged_variants(code):
    """(conv_tc lines, wgrad_tc lines) the launchers log while a child process runs `code` (python), each line as a dict of its
    integer fields, its output size (H, W) and the case `code` last named in a 'CASE <id>' line on stderr, in launch order"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, XUNET_CONV_LOG='1')
    r = subprocess.run([sys.executable, '-c', code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    conv, wgrad, case = [], [], None
    for line in r.stderr.splitlines():
        if line.startswith('CASE '):
            case = line[5:]
            continue
        kv = {k: int(v) for k, v in re.findall(r'(\w+)=(-?\d+)', line)}
        hw = re.search(r' (\d+)x(\d+) ', line)
        if hw:
            kv['H'], kv['W'] = int(hw.group(1)), int(hw.group(2))
        kv['case'] = case
        if line.startswith('conv_tc mode='):
            conv.append(kv)
        elif line.startswith('wgrad_tc '):
            wgrad.append(kv)
    return conv, wgrad


def test_tensor_core_variants_reached(lib):
    conv, wgrad = logged_variants('from tests.test_gpu_plan_launches import _launch_all_convs; _launch_all_convs()')
    reached = {
        'BN 32': any(c['BN'] == 32 for c in conv),
        'BN 64': any(c['BN'] == 64 for c in conv),
        'BN 128': any(c['BN'] == 128 for c in conv),
        'halo': any(c['halo'] == 1 for c in conv),
        'no halo': any(c['halo'] == 0 for c in conv),
        'one CTA per SM': any(c['per_sm'] == 1 for c in conv),
        'two CTAs per SM': any(c['per_sm'] == 2 for c in conv),
        'persistent grid, more tiles than CTAs': any(c['tiles'] > c['ctas'] for c in conv),
        'TMA reduce-add data gradient': any(c['mode'] == 1 and c['acc'] == 1 and c['tma_store'] == 1 for c in conv),
        'wgrad_tc with ksplit > 1': any(w['ksplit'] > 1 for w in wgrad),
    }
    print(f'{len(conv)} conv_tc and {len(wgrad)} wgrad_tc launches logged')
    print('conv_tc (mode, epi, BN, bk, halo, per_sm, acc, tma_store) seen:',
          sorted({(c['mode'], c['epi'], c['BN'], c['bk'], c['halo'], c['per_sm'], c['acc'], c['tma_store']) for c in conv}))
    print('wgrad_tc (BN, ksplit) seen:', sorted({(w['BN'], w['ksplit']) for w in wgrad}))
    for k, v in reached.items():
        print(f'  {k}: {"reached" if v else "NOT reached"}')
    assert all(reached.values()), [k for k, v in reached.items() if not v]
