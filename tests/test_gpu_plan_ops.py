"""Every conditioning, resampling, concat, attention-residual and loss op of the plans bench.py measures, element by element
against fp64 (tests/plan_ops_ref.py).

The op list comes from the plans themselves (xunet_plan_op), deduplicated by everything that changes a launch, plus three plans
that reach the pose-embedding paths bench.py's plans do not: SMALL at 64 with pos_emb and ref_pose_emb (bf16 at B = 8, fp32 at
B = 2) and SMALL with the opencv_uv ray convention.  Each op runs its forward and, in training plans, its backward through the
operator-level entry points at the plan's arguments, with a non-zero prior wherever the plan accumulates and garbage wherever it
overwrites.  Off-plan edges follow where the kernels branch: a partial last pixel block (S = 20), C / 4 odd, E from 4 to 2048,
B = 1 and 8, log-SNR beyond the clip, mixed cond_mask with and without explicit rays, |t| up to 8 and a skewed K, a zero loss.
Each check prints the worst err / bound and the element where it occurs.  The fp64 references run on the GPU."""
import dataclasses
import math

import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from tests import launch_ref as L
from tests import plan_ops_ref as O
from tests.test_gpu_plan_launches import DT, F64, _check, _gen, _offsets, _q, _rand, _s

pytestmark = pytest.mark.gpu

def _op_key(dtype, training, o):
    return (dtype, training) + tuple(o[k] for k in O.OP_KEY)


POSE_PLANS = {
    'small64_posemb': (dataclasses.replace(P.SMALL, use_pos_emb=True, use_ref_pose_emb=True), 64, 8, 1, 1),
    'small64_posemb_f32': (dataclasses.replace(P.SMALL, use_pos_emb=True, use_ref_pose_emb=True), 64, 2, 0, 1),
    'small64_opencv': (dataclasses.replace(P.SMALL, ray_convention='opencv_uv'), 64, 8, 1, 1),
}


def _unique_ops(lib, plans=None, exclude=None):
    """every op of `plans` (name -> (preset name or XUNetConfig, side, batch, dtype, training); default launch_ref.PLANS and
    POSE_PLANS) once, deduplicated by what changes its launches: [(id, dtype, training, op)].  Ops that the plans of `exclude`
    also have are left out."""
    if plans is None:
        plans = dict(L.PLANS, **POSE_PLANS)
    seen, out = set(), []
    if exclude is not None:
        seen.update(_op_key(dtype, training, o) for _, dtype, training, o in _unique_ops(lib, exclude))
    for plan, (cfg, S, B, dtype, training) in plans.items():
        for i, o in enumerate(O.plan_ops(lib, L.plan_config(cfg), B, S, dtype, training)):
            key = _op_key(dtype, training, o)
            if key in seen:
                continue
            seen.add(key)
            out.append((f'{plan}:op{i}', dtype, training, o))
    return out


UNIQUE = _unique_ops(_lib.load())


def _cases(kind):
    return [u for u in UNIQUE if u[3]['kind'] == kind]


def _ids(cases):
    return [c[0] for c in cases]


def _ok(lib, rc):
    assert rc == 0, lib.xunet_last_error()
    torch.cuda.synchronize()


def _p(t):
    return None if t is None else t.data_ptr()


# ======================================================================================================================
# log-SNR MLP
# ======================================================================================================================
def _run_logsnr(lib, name, B, E, backward):
    g = _gen(name)
    l = (torch.randn(B, generator=g, dtype=F64) * 8.).float()
    l[0] = -24.5                    # beyond the clip on both sides
    if B > 1:
        l[1] = 23.
    l = l.cuda()
    w0, w1 = (_rand((E, E), g, 1 / math.sqrt(E)).float() for _ in range(2))
    b0, b1 = (_rand((E,), g, 0.3).float() for _ in range(2))
    pe, h1, lemb = (torch.full((B, E), float('nan'), device='cuda') for _ in range(3))
    _ok(lib, lib.xunet_op_logsnr_emb(_p(l), _p(w0), _p(b0), _p(w1), _p(b1), _p(pe), _p(h1), _p(lemb), B, E, _s()))
    d = lambda t: t.to(F64)
    for what, ref, bound in O.logsnr_fwd_check(d(l), d(w0), d(b0), d(w1), d(b1), d(pe), d(h1)):
        _check(name, what, {'pe': pe, 'h1': h1, 'lemb': lemb}[what], ref, bound)
    if not backward:
        return
    dl = (_rand((B, E), g) + 0.2).float()
    for acc in (0, 1):
        priors = [_rand(s, g, 0.1).float() for s in ((E, E), (E,), (E, E), (E,))]
        outs = [p.clone() for p in priors]
        dh1 = torch.full((B, E), float('nan'), device='cuda')
        _ok(lib, lib.xunet_op_logsnr_emb_bwd(_p(dl), _p(w1), _p(pe), _p(h1), _p(dh1), *(_p(t) for t in outs), B, E, acc, _s()))
        got = dict(zip(('dh1', 'dw0', 'db0', 'dw1', 'db1'), [dh1] + outs))
        for what, ref, bound in O.logsnr_bwd_check(d(dl), d(w1), d(pe), d(h1), d(dh1), [d(p) for p in priors] if acc else None):
            _check(name, f'{what} (accumulate={acc})', got[what], ref, bound)


@pytest.mark.parametrize('case', _cases(_lib.PLAN_OP_LOGSNR), ids=_ids(_cases(_lib.PLAN_OP_LOGSNR)))
def test_logsnr_op(lib, case):
    name, dtype, training, o = case
    _run_logsnr(lib, name, o['B'], o['E'], training)


@pytest.mark.parametrize('B,E', [(1, 1024), (8, 1024), (8, 4), (1, 2048), (3, 96)])
def test_logsnr_edges(lib, B, E):
    _run_logsnr(lib, f'logsnr B={B} E={E}', B, E, True)


# ======================================================================================================================
# pose embedding
# ======================================================================================================================
def _cams(B, g):
    """rotations, centres up to |t| = 8 (position-channel arguments near 2^14 * 8 = 1.3e5), and intrinsics with cx != cy and a
    non-zero skew, all fp32 values"""
    q, _ = torch.linalg.qr(torch.randn(B, 3, 3, generator=g, dtype=F64))
    t = (torch.rand(B, 3, generator=g, dtype=F64) * 16. - 8.)
    t[0, 0] = 8.
    K = torch.tensor([[70., 0.7, 30.], [0., 65., 34.], [0., 0., 1.]], dtype=F64).repeat(B, 1, 1)
    K[:, 0, 0] += torch.rand(B, generator=g, dtype=F64)
    return [v.float().contiguous().cuda() for v in (q, t, K)]   # qr returns a column-major q


def _run_pose(lib, name, dtype, B, S, convention, pos_emb, ref_pose, backward, explicit_rays=False):
    g = _gen(name)
    R1, t1, K = _cams(B, g)
    R2, t2, _ = _cams(B, g)
    cond = torch.tensor([float(b % 3 != 1) for b in range(B)], device='cuda')     # mixed: samples 1, 4, 7 masked
    rays = None
    if explicit_rays:
        pos = torch.randn(B, 2, S, S, 3, generator=g, dtype=F64) * 3.
        dr = torch.randn(B, 2, S, S, 3, generator=g, dtype=F64)
        rays = torch.cat([pos, dr / dr.norm(dim=-1, keepdim=True)], -1).float().cuda()
    kinv = torch.full((B, 9), float('nan'), device='cuda')
    f64 = lambda t: None if t is None else t.to(F64)

    def run(pe, rf, ro):
        out = _rand((2 * B, S, S, 144), g).to(DT[dtype])     # garbage: every element is written
        _ok(lib, lib.xunet_op_pose_emb(dtype, _p(R1), _p(t1), _p(R2), _p(t2), _p(K), _p(cond), _p(pe), _p(rf), _p(ro),
                                       None if explicit_rays else _p(kinv), _p(out), B, S, convention, _p(rays), _s()))
        return out

    base = run(None, None, None)
    if not explicit_rays:
        ref, bound = O.kinv_check(K.to(F64).reshape(B, 9))
        _check(name, 'kinv', kinv, ref, bound)
    masked = (cond == 0).repeat_interleave(2)
    assert not base[masked].to(F64).any(), f'{name}: a masked sample is not 0'
    args = (dtype, f64(R1), f64(t1), f64(R2), f64(t2), f64(kinv), f64(cond), S, convention)
    dirs32 = None
    if dtype == 0 and not explicit_rays:
        # fp32: the directions the kernel stored (channels 93..95) against fp64 rays, then every channel at those directions
        dirs32 = base.to(F64).reshape(B, 2, S, S, 144)[..., 93:96]
        for f, Rf in enumerate((R1, R2)):
            d, de = O.ray_dirs(f64(kinv), f64(Rf), S, convention)
            on = cond != 0
            _check(name, f'directions of frame {f}', dirs32[on, f], d[on], de.expand_as(d)[on])
    ref, bound = O.pose_emb_check(*args, rays=f64(rays), dirs32=dirs32)
    _check(name, 'pose_emb', base, ref, bound)
    if pos_emb or ref_pose:
        pe = _rand((S, S, 144), g, 0.5).float() if pos_emb else None
        rf, ro = (_rand((144,), g, 0.5).float() for _ in range(2)) if ref_pose else (None, None)
        out = run(pe, rf, ro)
        # masked samples are exactly pos_emb + ref
        if dtype == 0:
            ex = O.pose_emb_added(dtype, base, pe, rf, ro)
            assert torch.equal(out, ex), f'{name}: pose_emb + pos_emb + ref is not the exact fp32 sum'
            print(f'{name} pose_emb with pos_emb / ref: bit-exact')
        else:
            ex = O.pose_emb_added(dtype, torch.zeros_like(base, dtype=torch.float32), pe, rf, ro)
            assert torch.equal(out[masked], ex[masked]), f'{name}: a masked sample is not exactly pos_emb + ref'
            ref, bound = O.pose_emb_check(*args, f64(pe), f64(rf), f64(ro), rays=f64(rays))
            _check(name, 'pose_emb with pos_emb / ref', out, ref, bound)
    if not backward:
        return
    dpose = (_rand((2 * B, S, S, 144), g) + _offsets(2 * B, 144)).to(DT[dtype])
    for acc in (0, 1):
        prior = _rand((S, S, 144), g).float()
        dpos = prior.clone()
        pr = [_rand((144,), g).float() for _ in range(2)]
        drf, dro = (p.clone() for p in pr)
        _ok(lib, lib.xunet_op_pose_emb_bwd(dtype, _p(dpose), _p(dpos), _p(drf) if ref_pose else None, _p(dro) if ref_pose else None,
                                           B, S, acc, _s()))
        ex, s0, s1 = O.pose_emb_bwd_exact(dpose, prior if acc else None)
        assert torch.equal(dpos, ex), f'{name}: dpos_emb (accumulate={acc}) is not the exact fp32 sum'
        print(f'{name} dpos_emb (accumulate={acc}): bit-exact')
        if ref_pose:
            for what, got, s, p in (('dref_first', drf, s0, pr[0]), ('dref_other', dro, s1, pr[1])):
                ref, bound = O.pose_emb_ref_check(s, p.to(F64))
                _check(name, what, got, ref, bound)


@pytest.mark.parametrize('case', _cases(_lib.PLAN_OP_POSE), ids=_ids(_cases(_lib.PLAN_OP_POSE)))
def test_pose_op(lib, case):
    name, dtype, training, o = case
    _run_pose(lib, name, dtype, o['B'], o['S'], o['ray_convention'], o['pos_emb'], o['ref_pose_emb'], o['need_grad'])


@pytest.mark.parametrize('dtype', [0, 1])
@pytest.mark.parametrize('convention,rays', [(0, False), (1, False), (0, True)], ids=['v3d130_ij', 'opencv_uv', 'explicit'])
def test_pose_edges(lib, dtype, convention, rays):
    """S = 20: 400 pixels, a partial last 64-pixel block; with pos_emb, ref and their gradients"""
    _run_pose(lib, f'pose S=20 dtype={dtype} conv={convention} rays={rays}', dtype, 3, 20, convention, True, True, True, rays)


# ======================================================================================================================
# FiLM embedding swish(lemb + pose-embedding level)
# ======================================================================================================================
def _run_film_emb(lib, name, dtype, N, HW, E, backward, write_dpe=True):
    g = _gen(name)
    bf = dtype == 1
    lemb = _rand((N // 2, E), g).float()
    pe = _q(_rand((N, HW, 1, E), g) + _offsets(N, E), dtype).reshape(N, HW, E)
    ped = pe.to(DT[dtype])
    semb = _rand((N, HW, E), g).to(DT[dtype])
    _ok(lib, lib.xunet_op_film_emb(dtype, _p(lemb), _p(ped), _p(semb), N, HW, E, _s()))
    ref, bound = O.film_emb_check(lemb.to(F64), pe, bf)
    _check(name, 'semb', semb, ref, bound)
    if not backward:
        return
    ds = _q(_rand((N, HW, 1, E), g) + _offsets(N, E), dtype).reshape(N, HW, E)
    prior = _rand((N // 2, E), g).float()
    dlemb = prior.clone()
    dpe0 = _rand((N, HW, E), g).to(DT[dtype])
    dpe = dpe0.clone()
    _ok(lib, lib.xunet_op_film_emb_bwd(dtype, _p(lemb), _p(ped), _p(ds.to(DT[dtype])), _p(dpe), _p(dlemb), N, HW, E, int(write_dpe),
                                       _s()))
    rdz, bdz, rdl, bdl = O.film_emb_bwd_check(lemb.to(F64), pe, ds, bf, prior.to(F64))
    if write_dpe:
        _check(name, 'dpe', dpe, rdz, bdz)
    else:
        assert torch.equal(dpe, dpe0)
    _check(name, 'dlemb', dlemb, rdl, bdl)


@pytest.mark.parametrize('case', _cases(_lib.PLAN_OP_EMB), ids=_ids(_cases(_lib.PLAN_OP_EMB)))
def test_film_emb_op(lib, case):
    name, dtype, training, o = case
    assert o['acc_x'] == 0
    _run_film_emb(lib, name, dtype, o['N'], o['H'] * o['W'], o['C'], training, o['write_dpe'])


@pytest.mark.parametrize('dtype', [0, 1])
@pytest.mark.parametrize('E', [4, 32, 96, 1024, 2048])
def test_film_emb_edges(lib, dtype, E):
    """E = 4, 32, 96: one to 24 threads per pixel (lane folding, idle threads); 1024: 256 threads; 2048: two passes"""
    _run_film_emb(lib, f'emb E={E} dtype={dtype}', dtype, 4, 400, E, True)


# ======================================================================================================================
# resample, concat copies, scale-add
# ======================================================================================================================
def _run_resample(lib, name, dtype, N, H, W, C, fwd, bwd, acc):
    """fwd = (pool, scale) on x (N, H, W, C); bwd = (pool, scale) on the output's gradient into a prior when acc, or None"""
    g = _gen(name)
    bf = dtype == 1
    pool, scale = fwd
    Ho, Wo = (H // 2, W // 2) if pool else (2 * H, 2 * W)
    x = _q(_rand((N, H, W, C), g) + _offsets(N, C), dtype)
    y = _rand((N, Ho, Wo, C), g).to(DT[dtype])
    _ok(lib, lib.xunet_op_resample(dtype, _p(x.to(DT[dtype])), _p(y), N, H, W, C, pool, scale, 0, _s()))
    ref, bound = O.resample_check(x, pool, scale, bf)
    _check(name, 'forward', y, ref, bound)
    if bwd is None:
        return
    bpool, bscale = bwd
    dy = _q(_rand((N, Ho, Wo, C), g) + _offsets(N, C), dtype)
    prior = _q(_rand((N, H, W, C), g) + _offsets(N, C), dtype)
    dx = prior.to(DT[dtype])
    _ok(lib, lib.xunet_op_resample(dtype, _p(dy.to(DT[dtype])), _p(dx), N, Ho, Wo, C, bpool, bscale, acc, _s()))
    ref, bound = O.resample_check(dy, bpool, bscale, bf, prior if acc else None)
    _check(name, f'backward (accumulate={acc})', dx, ref, bound)


@pytest.mark.parametrize('case', _cases(_lib.PLAN_OP_RESAMPLE), ids=_ids(_cases(_lib.PLAN_OP_RESAMPLE)))
def test_resample_op(lib, case):
    name, dtype, training, o = case
    _run_resample(lib, name, dtype, o['N'], o['H'], o['W'], o['C'], (o['fwd_pool'], o['fwd_scale']),
                  (o['bwd_pool'], o['bwd_scale']) if o['need_grad'] else None, o['acc_x'])


@pytest.mark.parametrize('dtype', [0, 1])
@pytest.mark.parametrize('rs', [_lib.RS_DOWN, _lib.RS_UP])
@pytest.mark.parametrize('acc', [0, 1])
def test_resample_edges(lib, dtype, rs, acc):
    """C = 36 (C / 4 odd): tail threads; the alias scale 1 / sqrt(2) on the backward"""
    down = rs == _lib.RS_DOWN
    gs = 1 / math.sqrt(2)
    _run_resample(lib, f'resample rs={rs} acc={acc} dtype={dtype}', dtype, 4, 10, 6, 36, (1, 0.25) if down else (0, 1.),
                  (0, 0.25 * gs) if down else (1, gs), acc)


def _run_concat(lib, name, dtype, npix, ca, cb, copies, acc_x, acc_r, backward):
    g = _gen(name)
    dt = DT[dtype]
    a, b = _rand((npix, ca), g).to(dt), _rand((npix, cb), g).to(dt)
    y = _rand((npix, ca + cb), g).to(dt)
    for src, cp in ((a, copies[0]), (b, copies[1])):
        _ok(lib, lib.xunet_op_copy_channels(dtype, _p(src), _p(y), npix, *cp, 0, _s()))
    assert torch.equal(y, torch.cat([a, b], -1)), f'{name}: the forward concat is not exact'
    if not backward:
        print(f'{name} forward copies: bit-exact')
        return
    dy = _rand((npix, ca + cb), g).to(dt)
    for k, (c, cp, acc) in enumerate(((ca, copies[2], acc_x), (cb, copies[3], acc_r))):
        prior = _rand((npix, c), g).to(dt)
        d = prior.clone()
        _ok(lib, lib.xunet_op_copy_channels(dtype, _p(dy), _p(d), npix, *cp, acc, _s()))
        assert torch.equal(d, O.copy_channels_exact(dy, prior, *cp, acc)), f'{name}: backward copy {k} (accumulate={acc}) not exact'
    print(f'{name} forward and backward copies: bit-exact')


@pytest.mark.parametrize('case', _cases(_lib.PLAN_OP_CONCAT), ids=_ids(_cases(_lib.PLAN_OP_CONCAT)))
def test_concat_op(lib, case):
    name, dtype, training, o = case
    _run_concat(lib, name, dtype, o['N'] * o['H'] * o['W'], o['C'], o['C2'], o['copies'], o['acc_x'], o['acc_r'],
                o['need_grad'] and o['need_grad_r'])


@pytest.mark.parametrize('dtype', [0, 1])
def test_concat_edges(lib, dtype):
    """C / 4 odd on both inputs, every copy accumulating into a prior"""
    ca, cb = 36, 20
    cps = ((ca, ca + cb, 0, 0, ca), (cb, ca + cb, 0, ca, cb), (ca + cb, ca, 0, 0, ca), (ca + cb, cb, ca, 0, cb))
    _run_concat(lib, f'concat 36+20 dtype={dtype}', dtype, 999, ca, cb, cps, 1, 1, True)
    # an accumulating copy into a destination offset (the forward layout)
    g = _gen(f'concat offset {dtype}')
    src = _rand((77, cb), g).to(DT[dtype])
    dst = _rand((77, ca + cb), g).to(DT[dtype])
    got = dst.clone()
    _ok(lib, lib.xunet_op_copy_channels(dtype, _p(src), _p(got), 77, *cps[1], 1, _s()))
    assert torch.equal(got, O.copy_channels_exact(src, dst, *cps[1], 1))


def _run_scale_add(lib, name, dtype, n, alpha, acc):
    g = _gen(name)
    bf = dtype == 1
    src = _q(_rand((n,), g), dtype)
    prior = _q(_rand((n,), g), dtype)
    dst = prior.to(DT[dtype])
    _ok(lib, lib.xunet_op_scale_add(dtype, _p(src.to(DT[dtype])), _p(dst), n, alpha, acc, _s()))
    ref, bound = O.scale_add_check(src, float(torch.tensor(alpha, dtype=torch.float32)), bf, prior if acc else None)
    _check(name, f'scale_add (accumulate={acc})', dst, ref, bound)


@pytest.mark.parametrize('case', _cases(_lib.PLAN_OP_ATTN_RESIDUAL), ids=_ids(_cases(_lib.PLAN_OP_ATTN_RESIDUAL)))
def test_attn_residual_op(lib, case):
    name, dtype, training, o = case
    if not o['need_grad']:
        pytest.skip('the residual gradient is added inside the GroupNorm backward (fused)')
    _run_scale_add(lib, name, dtype, o['N'] * o['H'] * o['W'] * o['C'], o['alpha'], o['acc_r'])


@pytest.mark.parametrize('dtype', [0, 1])
@pytest.mark.parametrize('acc', [0, 1])
def test_scale_add_edges(lib, dtype, acc):
    _run_scale_add(lib, f'scale_add dtype={dtype} acc={acc}', dtype, 4 * 1001, 1 / math.sqrt(2), acc)


# ======================================================================================================================
# loss
# ======================================================================================================================
def _run_loss(lib, name, dtype, B, S, zero=False):
    g = _gen(name)
    bf = dtype == 1
    eps = _rand((B, S, S, 3), g).float()
    noise = eps.clone() if zero else _rand((B, S, S, 3), g).float()
    sumsq, loss = torch.full((1,), 7., device='cuda'), torch.full((1,), 7., device='cuda')
    dO = _rand((2 * B, S, S, 3), g).to(DT[dtype])
    _ok(lib, lib.xunet_op_loss(dtype, _p(eps), _p(noise), _p(sumsq), _p(loss), _p(dO), B, S, _s()))
    ss, bss, lo, bl, rdo, bdo = O.loss_check(eps.to(F64), noise.to(F64), bf)
    _check(name, 'sumsq', sumsq, ss.reshape(1), bss.reshape(1))
    _check(name, 'loss', loss, lo.reshape(1), bl.reshape(1))
    _check(name, 'dO', dO, rdo, bdo)
    if zero:
        assert float(loss) == 0. and not dO.to(F64).isnan().any() and not dO.to(F64).any()


@pytest.mark.parametrize('case', _cases(_lib.PLAN_OP_LOSS), ids=_ids(_cases(_lib.PLAN_OP_LOSS)))
def test_loss_op(lib, case):
    name, dtype, training, o = case
    if not training:
        pytest.skip('no loss in a sampler plan')
    _run_loss(lib, name, dtype, o['B'], o['S'])


@pytest.mark.parametrize('dtype', [0, 1])
def test_loss_of_zero(lib, dtype):
    """eps_hat == eps: loss 0 gives dO = 0, not NaN"""
    _run_loss(lib, f'loss zero dtype={dtype}', dtype, 2, 20, zero=True)


# the check of each op kind, for op lists built from other plans (tests/test_gpu_plan_sweep.py)
OP_CHECKS = {_lib.PLAN_OP_LOGSNR: test_logsnr_op, _lib.PLAN_OP_POSE: test_pose_op, _lib.PLAN_OP_EMB: test_film_emb_op,
             _lib.PLAN_OP_RESAMPLE: test_resample_op, _lib.PLAN_OP_CONCAT: test_concat_op,
             _lib.PLAN_OP_ATTN_RESIDUAL: test_attn_residual_op, _lib.PLAN_OP_LOSS: test_loss_op}
