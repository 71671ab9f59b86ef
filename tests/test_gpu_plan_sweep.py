"""The conv, attention and conditioning launches of plans beyond the benchmarked ones, element by element against fp64, and a
table of the kernel variants they reach.

tests/test_gpu_plan_launches.py and tests/test_gpu_plan_ops.py check the launches of the plans bench.py measures: B in {2, 4,
8}, sides that are powers of two, square images.  xunet_create accepts much more (any batch, any side divisible by
2^(levels - 1), ch a multiple of 32, head_dim 16 to 128), and the launchers pick a kernel and its variant from the shape.  SWEEP
lists plans chosen for the branches they reach:
  * batch 1, 2, 3, 5 next to 4 and 8: an odd N / 2 changes whether a tile of frames divides N, and every grid and split-K;
  * sides 16 and 32, where the deep configurations reach the 4 x 4 and 2 x 2 levels; 24, 48 and 96, which send every bf16 conv
    to the SIMT kernels and attention to L = 576, 144 and 36; 18, where the three-channel direct kernels meet W % 4 != 0; 256,
    where a 128-pixel row tile spans half a row;
  * ch 96 and 160 (Ci of 96 to 480 through the skip concats, Co / 32 odd) and head_dim 16, 32, 64 and 128 on both attention
    kernels; pos_emb and ref_pose_emb on and off; training and sampling plans; fp32 plans.
Their launches, minus those of the benchmarked plans and one per class of kernels and shape (_one_per_class), run through the
same checks as the benchmarked plans' (check_conv, check_attention, OP_CHECKS).  Operator-level cases (OP_CONVS) add what no
model configuration reaches, and non-square images for the tensor-core conv and weight gradient.

test_variant_coverage runs every checked conv launch once more in a child process that logs the tensor-core launchers' choices
(XUNET_CONV_LOG), and fails when a variant of VARIANTS is reached by none; the printed table names the launch each variant was
checked on."""
import ctypes
import dataclasses

import pytest

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from tests import launch_ref as L
from tests.test_gpu_plan_launches import ATTNS as BENCH_ATTNS, CONVS as BENCH_CONVS, check_attention, check_conv, logged_variants
from tests.test_gpu_plan_ops import OP_CHECKS, POSE_PLANS, _unique_ops

pytestmark = pytest.mark.gpu

_C = lambda **kw: dataclasses.replace(P.SMALL, **kw)
# name -> (XUNetConfig, side, xunet_create batch, dtype (0 fp32, 1 bf16), training)
SWEEP = {
    # 16 x 16 and 8 x 8 at N = 2: head_dim 16 on the tensor cores (L = 256), 32 on the SIMT kernel (L = 64)
    'tiny16_b1': (_C(ch=32, ch_mult=(1, 2), attn_resolutions=(16, 8), attn_heads=2), 16, 1, 1, 1),
    # down to 2 x 2: at 4 x 4 a tile holds 8 frames, which N = 6 / 10 does not divide (SIMT); N = 8 does (tensor cores)
    'deep16_b3_s': (_C(ch=32, ch_mult=(1, 2, 2, 4), attn_resolutions=(16, 8, 4), attn_heads=2), 16, 3, 1, 0),
    'deep16_b5': (_C(ch=32, ch_mult=(1, 2, 2, 4), attn_resolutions=(16, 8), attn_heads=2, use_pos_emb=True), 16, 5, 1, 1),
    'full16_b4': (P.FULL_3DIM, 16, 4, 1, 1),
    'full32_b2': (P.FULL_3DIM, 32, 2, 1, 1),
    'full32_b2_s': (P.FULL_3DIM, 32, 2, 1, 0),
    # sides 128 neither divides nor is a multiple of: every bf16 conv and attention on the SIMT kernels
    'side24_b2': (_C(ch=64, ch_mult=(1, 2, 4), attn_resolutions=(24, 12, 6), attn_heads=2, use_ref_pose_emb=True), 24, 2, 1, 1),
    'side48_b1': (_C(ch=32, ch_mult=(1, 2, 2, 4), attn_resolutions=(12, 6), attn_heads=1), 48, 1, 1, 1),
    'side96_b1_s': (_C(ch=32, ch_mult=(1, 2, 2, 4), attn_resolutions=(12,), attn_heads=2), 96, 1, 1, 0),
    'side18_b2': (_C(ch=32, ch_mult=(1, 2), attn_resolutions=()), 18, 2, 1, 1),
    'small256_b1': (P.SMALL, 256, 1, 1, 1),
    # Co / 32 odd: 32-wide dY blocks and BN = 32 in the weight gradient, BN = 32 in the conv
    'ch96_b2': (_C(ch=96, ch_mult=(1, 2, 3), attn_resolutions=(16,), attn_heads=6, use_pos_emb=True, use_ref_pose_emb=True), 32, 2, 1,
                1),
    'ch160_b3': (_C(ch=160, ch_mult=(1, 2, 4), attn_resolutions=(8,), attn_heads=5), 32, 3, 1, 1),
    'ch160_b8_s': (_C(ch=160, ch_mult=(1, 2, 4), attn_resolutions=(16,), attn_heads=10), 32, 8, 1, 0),
    'f32_deep16_b1': (_C(ch=32, ch_mult=(1, 2, 2), attn_resolutions=(16, 8, 4), attn_heads=1), 16, 1, 0, 1),
    'f32_ch96_b3': (_C(ch=96, ch_mult=(1, 2), attn_resolutions=(16, 8), attn_heads=3, use_pos_emb=True, use_ref_pose_emb=True), 16, 3,
                    0, 1),
    'f32_side24_b2_s': (_C(ch=64, ch_mult=(1, 2), attn_resolutions=(24, 12), attn_heads=1), 24, 2, 0, 0),
    'f32_side18_b1': (_C(ch=32, ch_mult=(1, 2), attn_resolutions=()), 18, 1, 0, 1),
    'f32_side48_b1': (_C(ch=32, ch_mult=(1, 2), attn_resolutions=()), 48, 1, 0, 1),
}
WORKSPACE_LIMIT = 8 << 30       # each plan's activations and gradients; the checks below allocate far less


def _tc(r):
    return _lib.KERNEL_TC in (r['fwd'], r['dgrad'], r['wgrad'])


def _class(dtype, training, r):
    """launches of one class reach the same kernel variants: the kernels, the epilogue and the shape they are chosen by.  A
    tensor-core launch's tiling and split follow H, W, N and the channel residues; a SIMT or direct kernel's only W's."""
    if r['kind'] == 1:
        return (1, dtype, training, r['N'] % 4 == 0, r['L'], r['C'] // r['heads'], r['cross'], r['impl'], r['emits_stats'])
    k = (0, dtype, training) + tuple(r[x] for x in ('fwd', 'dgrad', 'wgrad', 'ksize', 'stride', 'nseg', 'residual', 'emits_stats',
                                                    'gn_mode', 'accumulate'))
    if _tc(r):
        return k + (r['Ho'], r['Wo'], r['N'], r['Ci'] % 128, r['Co'] % 128)
    return k + (min(r['Wo'], 32), r['Wo'] % 32, r['Ci'] % 64, r['Co'] % 64)


def _op_class(dtype, training, o):
    """ops of one class take the same branches of their kernels: the op and its flags, the image size, the channel residues"""
    return (dtype, training) + tuple(o[k] for k in ('kind', 'S', 'H', 'W', 'rs', 'fwd_pool', 'bwd_pool', 'acc_x', 'acc_r', 'need_grad',
                                                    'need_grad_r', 'write_dpe', 'pos_emb', 'ref_pose_emb')) + (o['C'] % 8, o['C2'] % 8)


def _one_per_class(launches, key=_class):
    seen, out = set(), []
    for u in launches:
        k = key(u[1], u[2], u[3])
        if k not in seen:
            seen.add(k)
            out.append(u)
    return out


def _op_conv(name, N, H, W, Ci, Co, ks, dgrad=_lib.KERNEL_TC, **kw):
    """an operator-level conv case in the form of a plan launch (xunet_plan_launch's fields), checked by check_conv"""
    r = dict(kind=0, leaf=0, N=N, Hi=H, Wi=W, Ci=Ci, Ho=H, Wo=W, Co=Co, ksize=ks, stride=1, nseg=1, residual=0, alpha=1.,
             fwd=_lib.KERNEL_TC, dgrad=dgrad, wgrad=_lib.KERNEL_TC, emits_stats=0, bwd_alpha=1., accumulate=0, gn_mode=-1, L=0, C=0,
             heads=0, cross=0, impl=0)
    r.update(kw)
    return (f'op:{name}', 1, 1, r)


# Ci = 16 / 48: no model configuration has them (channels are multiples of 32, or the 144 pose-embedding channels); they reach
# the 16-wide K chunks of the conv and the CWA = 16 weight-gradient instances.  The data gradient's GEMM N (= Ci) is then not a
# multiple of 32, which sends it to the SIMT kernel.  The rest are non-square images: halo tiles (3 x 3, W % 16 == 0, H % 8 == 0)
# and plain ones, with the fused statistics and the TMA reduce-add data gradient.
OP_CONVS = [
    _op_conv('Ci48 Co64 16x16 3x3', 2, 16, 16, 48, 64, 3, dgrad=_lib.KERNEL_SIMT),
    _op_conv('Ci48 Co128 16x32 1x1', 2, 16, 32, 48, 128, 1, dgrad=_lib.KERNEL_SIMT, alpha=0.7071),
    _op_conv('Ci16 Co96 8x32 3x3', 2, 8, 32, 16, 96, 3, dgrad=_lib.KERNEL_SIMT, residual=1),
    _op_conv('halo 16x64 Ci64 Co64 stats acc', 2, 16, 64, 64, 64, 3, emits_stats=1, accumulate=1),
    _op_conv('halo 64x16 Ci32 Co128', 2, 64, 16, 32, 128, 3, residual=1, alpha=0.7071),
    _op_conv('halo 8x32 Ci96 Co64', 2, 8, 32, 96, 64, 3, bwd_alpha=0.5),
    _op_conv('rows 32x8 Ci64 Co64', 2, 32, 8, 64, 64, 3, residual=1),
    _op_conv('frames 4x16 Ci64 Co64', 4, 4, 16, 64, 64, 3, emits_stats=1),
    _op_conv('1x1 16x64 Ci64 Co128 acc', 2, 16, 64, 64, 128, 1, accumulate=1),
    _op_conv('1x1 64x16 Ci128 Co96', 2, 64, 16, 128, 96, 1),
]

_LIB = _lib.load()
UNIQUE = _one_per_class(L.unique_launches(_LIB, SWEEP, exclude=L.PLANS))
CONVS = [u for u in UNIQUE if u[3]['kind'] == _lib.LAUNCH_CONV] + OP_CONVS
ATTNS = [u for u in UNIQUE if u[3]['kind'] == _lib.LAUNCH_ATTN]
# a sampler plan runs no loss; an attention residual's gradient is its own launch only where the plan does not fuse it into the
# GroupNorm backward
OPS = [u for u in _one_per_class(_unique_ops(_LIB, SWEEP, exclude=dict(L.PLANS, **POSE_PLANS)), _op_class)
       if not (u[3]['kind'] == _lib.PLAN_OP_LOSS and not u[2]) and not (u[3]['kind'] == _lib.PLAN_OP_ATTN_RESIDUAL and not u[3]['need_grad'])]
PLANS = dict(L.PLANS, **SWEEP)


def _ids(cases):
    return [c[0] for c in cases]


@pytest.mark.parametrize('plan', list(SWEEP))
def test_sweep_plan_fits(lib, plan):
    cfg, S, B, dtype, training = SWEEP[plan]
    h = ctypes.c_void_p()
    cs = cfg.c_struct()
    assert lib.xunet_create(ctypes.byref(cs), B, S, dtype, training, ctypes.byref(h)) == 0, lib.xunet_last_error()
    try:
        ws = lib.xunet_workspace_bytes(h)
    finally:
        lib.xunet_destroy(h)
    print(f'{plan}: workspace {ws / 2 ** 20:.0f} MiB')
    assert 0 < ws < WORKSPACE_LIMIT


@pytest.mark.parametrize('case', CONVS, ids=_ids(CONVS))
def test_sweep_conv_launch(lib, case):
    check_conv(lib, case, PLANS)


@pytest.mark.parametrize('peaked', [False, True], ids=['moderate', 'peaked'])
@pytest.mark.parametrize('case', ATTNS, ids=_ids(ATTNS))
def test_sweep_attention_launch(lib, case, peaked):
    check_attention(lib, case, peaked)


@pytest.mark.parametrize('case', OPS, ids=_ids(OPS))
def test_sweep_op(lib, case):
    OP_CHECKS[case[3]['kind']](lib, case)


# ======================================================================================================================
# which variant each checked launch ran
# ======================================================================================================================
def _launch_checked_convs():
    """every conv launch test_conv_launch and test_sweep_conv_launch check, once more on zero-filled buffers, each after a
    'CASE <id>' line on stderr (the child of test_variant_coverage)"""
    import sys
    from tests.test_gpu_plan_launches import _launch_all_convs
    for case in BENCH_CONVS + CONVS:
        print(f'CASE {case[0]}', file=sys.stderr, flush=True)
        _launch_all_convs([case])


def _K(c):
    """the GEMM reduction channels per tap of a logged conv_tc launch"""
    return c['wCi'] if c['mode'] == 0 else c['segw']


def _Nn(c):
    return c['wCo'] if c['mode'] == 0 else c['wCi']


SIMT, TC, CIN3, COUT3, NONE = _lib.KERNEL_SIMT, _lib.KERNEL_TC, _lib.KERNEL_CIN3, _lib.KERNEL_COUT3, _lib.KERNEL_NONE
_ANY = lambda r, k: k in (r['fwd'], r['dgrad'], r['wgrad'])
_NOT_POW2_DIVISOR = lambda w: 128 % w != 0 and w % 128 != 0
_UNREACHABLE_C = 'no model configuration has 16 or 48 channels (multiples of 32, or the 144 pose-embedding channels)'

# (variant, where it is read (conv_tc / wgrad_tc log lines, or conv / attn plan launches), predicate, reason no model
# configuration reaches it (then an op: case must))
VARIANTS = [
    # conv_tc: pick_tile's tiles, and the halo re-tiling
    ('conv_tc rows of 128 pixels (W >= 128)', 'conv_tc', lambda c: c['halo'] == 0 and c['W'] >= 128, None),
    ('conv_tc whole rows (W < 128 <= H W)', 'conv_tc', lambda c: c['halo'] == 0 and c['W'] < 128 <= c['H'] * c['W'], None),
    ('conv_tc whole frames (H W < 128, TN > 1)', 'conv_tc', lambda c: c['halo'] == 0 and c['H'] * c['W'] < 128, None),
    ('conv_tc frames at 4 x 4 (TN = 8)', 'conv_tc', lambda c: c['H'] == 4 and c['W'] == 4, None),
    ('conv_tc halo tiles', 'conv_tc', lambda c: c['halo'] == 1, None),
    ('conv_tc halo tiles, H != W', 'conv_tc', lambda c: c['halo'] == 1 and c['H'] != c['W'], 'every model image is square'),
    ('conv_tc plain tiles, H != W', 'conv_tc', lambda c: c['halo'] == 0 and c['H'] != c['W'], 'every model image is square'),
    # pick_bk, with and without a zero-filled tail chunk, and the halo BK 64 -> 32 fallback
    ('conv_tc bk 64', 'conv_tc', lambda c: c['bk'] == 64 and _K(c) % 64 == 0, None),
    ('conv_tc bk 64 with a zero-filled tail', 'conv_tc', lambda c: c['bk'] == 64 and _K(c) % 64 != 0, None),
    ('conv_tc bk 32', 'conv_tc', lambda c: c['bk'] == 32 and _K(c) % 64 != 0, None),
    ('conv_tc bk 16', 'conv_tc', lambda c: c['bk'] == 16, _UNREACHABLE_C),
    ('conv_tc halo bk 64 -> 32', 'conv_tc', lambda c: c['halo'] == 1 and c['bk'] == 32 and _K(c) % 64 == 0, None),
    # BN, and its halving when the tiles do not fill the device
    ('conv_tc BN 32', 'conv_tc', lambda c: c['BN'] == 32, None),
    ('conv_tc BN 64', 'conv_tc', lambda c: c['BN'] == 64, None),
    ('conv_tc BN 128', 'conv_tc', lambda c: c['BN'] == 128, None),
    ('conv_tc BN halved for few tiles', 'conv_tc',
     lambda c: c['BN'] < (128 if _Nn(c) % 128 == 0 else 64 if _Nn(c) % 64 == 0 else 32), None),
    ('conv_tc one CTA per SM', 'conv_tc', lambda c: c['per_sm'] == 1, None),
    ('conv_tc two CTAs per SM', 'conv_tc', lambda c: c['per_sm'] == 2, None),
    ('conv_tc more tiles than CTAs', 'conv_tc', lambda c: c['tiles'] > c['ctas'], None),
    ('conv_tc ring shorter than 3 (steps < stages)', 'conv_tc', lambda c: c['stages'] < 3, None),
    ('conv_tc epilogue 0 (plain)', 'conv_tc', lambda c: c['epi'] == 0, None),
    ('conv_tc epilogue 1 (GroupNorm statistics)', 'conv_tc', lambda c: c['epi'] == 1, None),
    ('conv_tc epilogue 2 (GroupNorm backward)', 'conv_tc', lambda c: c['epi'] == 2, None),
    ('conv_tc epilogue 3 (GroupNorm + FiLM backward)', 'conv_tc', lambda c: c['epi'] == 3, None),
    ('conv_tc TMA reduce-add (accumulating data gradient)', 'conv_tc', lambda c: c['acc'] == 1 and c['tma_store'] == 1, None),
    ('conv_tc TMA store (1 x 1 forward)', 'conv_tc', lambda c: c['acc'] == 0 and c['tma_store'] == 1, None),
    ('conv_tc strided forward', 'conv_tc', lambda c: c['st'] > 1, None),
    ('conv_tc segmented data gradient (q|k|v)', 'conv_tc', lambda c: c['mode'] == 1 and c['segw'] != c['wCo'], None),
    # wgrad_tc: the template instances <CWA, CWB, BN>, the tail, the bias block, the split
    *[(f'wgrad_tc <{a}, {b}, {n}>', 'wgrad_tc', (lambda a, b, n: lambda w: (w['cwa'], w['cwb'], w['BN']) == (a, b, n))(a, b, n),
       _UNREACHABLE_C if a == 16 else None)
      for a in (64, 32, 16) for b, n in ((64, 128), (64, 64), (32, 32))],
    ('wgrad_tc zero-filled Ci tail', 'wgrad_tc', lambda w: w['Ci'] % w['cwa'] != 0, None),
    ('wgrad_tc bias block in its own M tile', 'wgrad_tc', lambda w: w['MB'] % (128 // w['cwa']) == 0, None),
    ('wgrad_tc bias block in the last weight tile', 'wgrad_tc', lambda w: w['MB'] % (128 // w['cwa']) != 0, None),
    ('wgrad_tc ksplit = 1', 'wgrad_tc', lambda w: w['ksplit'] == 1, None),
    ('wgrad_tc ksplit > 1', 'wgrad_tc', lambda w: w['ksplit'] > 1, None),
    ('wgrad_tc strided', 'wgrad_tc', lambda w: w['st'] > 1, None),
    ('wgrad_tc frames (H W < 128)', 'wgrad_tc', lambda w: w['H'] * w['W'] < 128, None),
    ('wgrad_tc H != W', 'wgrad_tc', lambda w: w['H'] != w['W'], 'every model image is square'),
    # the SIMT and direct kernels, read from the plan launch
    ('SIMT conv bf16, forward / data / weight gradient', 'conv',
     lambda d, r: d == 1 and r['fwd'] == SIMT and r['dgrad'] == SIMT and r['wgrad'] == SIMT, None),
    ('SIMT conv bf16 at a side 128 neither divides nor multiplies', 'conv',
     lambda d, r: d == 1 and r['fwd'] == SIMT and _NOT_POW2_DIVISOR(r['Wo']), None),
    ('SIMT conv bf16 at 4 x 4, N not a multiple of the 8-frame tile', 'conv',
     lambda d, r: d == 1 and r['fwd'] == SIMT and r['Ho'] == 4 and r['N'] % 8 != 0, None),
    ('SIMT conv fp32, forward / data / weight gradient', 'conv',
     lambda d, r: d == 0 and r['fwd'] == SIMT and r['dgrad'] == SIMT and r['wgrad'] == SIMT, None),
    ('SIMT conv, strided (pose embedding)', 'conv', lambda d, r: r['stride'] > 1 and r['fwd'] == SIMT, None),
    *[(f'{k} {dn}, {wn}', 'conv', (lambda kern, dt, wp: lambda d, r: d == dt and _ANY(r, kern) and wp(r['Wo']))(kern, dt, wp), None)
      for k, kern in (('cin3', CIN3), ('cout3', COUT3)) for dn, dt in (('bf16', 1), ('fp32', 0))
      for wn, wp in (('W % 32 == 0', lambda w: w % 32 == 0), ('W < 32, W % 4 == 0', lambda w: w < 32 and w % 4 == 0),
                     ('W > 32, W % 32 != 0', lambda w: w > 32 and w % 32 != 0 and w % 4 == 0), ('W % 4 != 0', lambda w: w % 4 != 0))],
    # attention: every head_dim on both kernels
    *[(f'attention {"tensor-core" if impl else "SIMT"} head_dim {hd}', 'attn',
       (lambda impl, hd: lambda d, tr, r: r['impl'] == impl and r['C'] // r['heads'] == hd)(impl, hd), None)
      for impl in (1, 0) for hd in (16, 32, 64, 128)],
    ('attention SIMT L % 32 != 0 (partial key chunk)', 'attn', lambda d, tr, r: r['impl'] == 0 and r['L'] % 32 != 0, None),
    ('attention SIMT L % 8 != 0', 'attn', lambda d, tr, r: r['impl'] == 0 and r['L'] % 8 != 0, None),
    ('attention SIMT backward, L % 128 != 0', 'attn', lambda d, tr, r: r['impl'] == 0 and tr and r['L'] % 128 != 0, None),
    ('attention SIMT bf16 (L % 128 != 0)', 'attn', lambda d, tr, r: r['impl'] == 0 and d == 1 and r['L'] % 128 != 0, None),
    ('attention tensor-core backward head_dim 16', 'attn', lambda d, tr, r: r['impl'] == 1 and tr and r['C'] // r['heads'] == 16,
     None),
]


def test_variant_coverage(lib):
    conv, wgrad = logged_variants('from tests.test_gpu_plan_sweep import _launch_checked_convs; _launch_checked_convs()')
    assert conv and wgrad and all(x['case'] for x in conv + wgrad)
    plan_convs = [(u[0], u[1], u[3]) for u in BENCH_CONVS + CONVS]
    plan_attns = [(u[0], u[1], u[2], u[3]) for u in BENCH_ATTNS + ATTNS]

    def first(where, pred):
        """the first checked launch that reaches the variant, and how many do ('mode' 0: conv forward, 1: data gradient)"""
        if where == 'conv_tc':
            hits = [f"{x['case']} (mode {x['mode']})" for x in conv if pred(x)]
        elif where == 'wgrad_tc':
            hits = [x['case'] for x in wgrad if pred(x)]
        elif where == 'conv':
            hits = [n for n, d, rr in plan_convs if pred(d, rr)]
        else:
            hits = [n for n, d, tr, rr in plan_attns if pred(d, tr, rr)]
        return (hits[0], len(hits)) if hits else (None, 0)

    missing = []
    print(f'\n{len(conv)} conv_tc and {len(wgrad)} wgrad_tc launches logged; {len(plan_convs)} conv and {len(plan_attns)} attention '
          'launches checked')
    width = max(len(v[0]) for v in VARIANTS)
    for name, where, pred, reason in VARIANTS:
        got, n = first(where, pred)
        seen = f'{got} and {n - 1} more' if got else 'NOT REACHED'
        if reason is None:
            print(f'  {name:<{width}}  {seen}')
            ok = got is not None
        else:
            print(f'  {name:<{width}}  {seen}  [no plan: {reason}]')
            ok = got is not None and got.startswith('op:')
        if not ok:
            missing.append(name)
    assert not missing, missing
