"""CPU checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/xunet_b200.h declares,
and its static plan (parameter tree, workspace) agrees with the oracle's walk of model/xunet.py.  No compute calls."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import xunet_ref as R
from tests import launch_ref as L
from novel_view_synthesis_3d_b200 import _lib, XUNetConfig, SMALL, FULL_3DIM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_all_exported(lib):
    hdr = open(os.path.join(ROOT, 'include', 'xunet_b200.h')).read()
    declared = set(re.findall(r'\b(xunet_[a-z_0-9]+)\s*\(', hdr))
    assert declared, 'no declarations parsed'
    assert declared == set(_lib.SYMBOLS), (declared ^ set(_lib.SYMBOLS))
    for name in declared:
        assert hasattr(lib, name)
    assert lib.xunet_version() >= 100


def _spec(lib, cfg: XUNetConfig, B, S, training=0, dtype=1):
    h = C.c_void_p()
    cs = cfg.c_struct()
    assert lib.xunet_create(C.byref(cs), B, S, dtype, training, C.byref(h)) == 0, lib.xunet_last_error()
    spec = {}
    name, ndim, shape, off = C.c_char_p(), C.c_int(), (C.c_longlong * 5)(), C.c_longlong()
    for i in range(lib.xunet_param_leaves(h)):
        assert lib.xunet_param_leaf(h, i, C.byref(name), C.byref(ndim), C.byref(shape), C.byref(off)) == 0
        spec[name.value.decode()] = (tuple(shape[k] for k in range(ndim.value)), off.value)
    n, ws = lib.xunet_param_count(h), lib.xunet_workspace_bytes(h)
    lib.xunet_destroy(h)
    return spec, n, ws


@pytest.mark.parametrize('cfg,S', [
    (SMALL, 64), (SMALL, 128), (FULL_3DIM, 128), (FULL_3DIM, 64),
    (XUNetConfig(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2,
                 use_pos_emb=True, use_ref_pose_emb=True), 16),
    (XUNetConfig(ch=64, ch_mult=(1, 2, 4), emb_ch=64, num_res_blocks=1, attn_resolutions=(8,), attn_heads=4), 32),
])
def test_param_tree_matches_flax_walk(lib, cfg, S):
    from tests.util import to_ref_cfg
    spec, n, ws = _spec(lib, cfg, 2, S)
    ref = R.param_shapes(to_ref_cfg(cfg), S)
    assert set(spec) == set(ref)
    for k, shp in ref.items():
        assert spec[k][0] == tuple(shp), k
    assert n == sum(int(np.prod(s)) for s in ref.values())
    # leaves tile the flat buffer exactly
    spans = sorted((off, off + int(np.prod(shp))) for shp, off in spec.values())
    assert spans[0][0] == 0 and spans[-1][1] == n
    assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
    assert ws > 0


def test_known_param_counts(lib):
    assert _spec(lib, SMALL, 1, 64)[1] == 1054211
    assert _spec(lib, SMALL, 1, 128)[1] == 902915
    assert _spec(lib, FULL_3DIM, 1, 128)[1] == 438831363
    assert _spec(lib, FULL_3DIM, 1, 64)[1] == 449877251


def test_create_rejects_bad_configs(lib):
    h = C.c_void_p()
    bad = [XUNetConfig(ch=48), XUNetConfig(emb_ch=30), XUNetConfig(dropout=1.0),
           XUNetConfig(ch=32, ch_mult=(1, 2), attn_heads=3)]
    for cfg in bad:
        cs = cfg.c_struct()
        assert lib.xunet_create(C.byref(cs), 2, 64, 1, 0, C.byref(h)) != 0
        assert lib.xunet_last_error()
    cs = SMALL.c_struct()
    assert lib.xunet_create(C.byref(cs), 2, 63, 1, 0, C.byref(h)) != 0      # side not divisible by 2^(L-1)
    assert lib.xunet_create(C.byref(cs), 2, 64, 7, 0, C.byref(h)) != 0      # bad dtype


def test_training_workspace_is_larger(lib):
    assert _spec(lib, SMALL, 2, 64, training=1)[2] > _spec(lib, SMALL, 2, 64, training=0)[2]
    assert _spec(lib, SMALL, 2, 64, dtype=0)[2] > _spec(lib, SMALL, 2, 64, dtype=1)[2]


def test_no_cpu_fallback():
    """The product path must fail loudly without a GPU (no eager / CPU fallback)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from novel_view_synthesis_3d_b200 import XUNet
    with pytest.raises(RuntimeError, match='CUDA device'):
        XUNet().engine(1, 64)


def test_library_is_built_from_the_sources_in_the_tree():
    """A stale or failed build must not go unnoticed (the .so is git-ignored and travels with the tree): build() is a no-op when
    the stamp matches the sources, recompiles otherwise, and raises on any nvcc error."""
    from novel_view_synthesis_3d_b200 import build as B
    lib = B.build()
    assert lib.exists()
    deps = list(B.CSRC.glob('*.cu')) + list(B.CSRC.glob('*.cuh')) + list(B.CSRC.glob('*.h')) + list(B.INCLUDE.glob('*.h'))
    assert (B.OBJ_DIR / 'stamp').read_text() == B._digest(deps)


# ---- the plan's conv and attention launches (xunet_plan_launch), for every plan bench.py measures ----
@pytest.mark.parametrize('plan', list(L.PLANS))
def test_plan_launches_cover_every_conv_leaf_and_attention_block(lib, plan):
    import novel_view_synthesis_3d_b200 as P
    from tests.util import to_ref_cfg
    preset, S, B, dtype, training = L.PLANS[plan]
    cfg = getattr(P, preset)
    launches, names = L.plan_launches(lib, cfg, B, S, dtype, training)
    ref = R.param_shapes(to_ref_cfg(cfg), S)
    convs = [r for r in launches if r['kind'] == _lib.LAUNCH_CONV]
    attns = [r for r in launches if r['kind'] == _lib.LAUNCH_ATTN]
    assert len(convs) + len(attns) == len(launches)
    # one conv per kernel leaf: every conv, 1x1 Dense and FiLM Dense, and the q|k|v projection (its q kernel leads the three
    # segments); the log-SNR MLP is not a conv
    conv_leaves = {n for n in ref if n.endswith('/kernel') and not n.startswith('ConditioningProcessor_0/Dense_') and
                   'DenseGeneral_1' not in n and 'DenseGeneral_2' not in n}
    got = [names[r['leaf']] for r in convs]
    assert sorted(got) == sorted(conv_leaves)
    for r in convs:
        shp = ref[names[r['leaf']]]
        if 'DenseGeneral_0' in names[r['leaf']]:
            ks, ci, co, nseg = 1, shp[0], 3 * shp[1] * shp[2], 3
        elif len(shp) == 5:
            ks, ci, co, nseg = shp[1], shp[3], shp[4], 1
        else:
            ks, ci, co, nseg = 1, shp[0], shp[1], 1
        assert (r['ksize'], r['Ci'], r['Co'], r['nseg']) == (ks, ci, co, nseg), names[r['leaf']]
        assert r['N'] == 2 * B
        if not training:
            assert r['dgrad'] == r['wgrad'] == _lib.KERNEL_NONE
        else:
            assert r['wgrad'] != _lib.KERNEL_NONE
        if r['gn_mode'] >= 0:
            assert r['dgrad'] == _lib.KERNEL_TC and not r['accumulate']
    # one attention per AttnBlock, in op order, with its C and heads
    blocks = [n[:-len('/AttnLayer_0/DenseGeneral_0/kernel')] for n in names if n.endswith('AttnLayer_0/DenseGeneral_0/kernel')]
    assert len(attns) == len(blocks)
    for r, b in zip(attns, blocks):
        C_, heads, hd = ref[b + '/AttnLayer_0/DenseGeneral_0/kernel']
        assert (r['C'], r['heads']) == (C_, heads) and C_ == heads * hd
        assert r['cross'] == int(b.endswith('AttnBlock_1'))
        # tensor cores in bf16 exactly for L a multiple of 128 and head_dim 16, 32, 64 or 128; never in fp32
        assert r['impl'] == int(dtype == 1 and r['L'] % 128 == 0 and hd in (16, 32, 64, 128)), (b, r)
    if dtype == 0:
        assert all(_lib.KERNEL_TC not in (r['fwd'], r['dgrad'], r['wgrad']) for r in convs)
        assert all(r['impl'] == 0 for r in attns)


# ---- the plan's other ops (xunet_plan_op): counts against the topology, the resample adjoints and their alias scales ----
@pytest.mark.parametrize('plan', list(L.PLANS))
def test_plan_ops_match_the_topology(lib, plan):
    import novel_view_synthesis_3d_b200 as P
    from tests import plan_ops_ref as O
    preset, S, B, dtype, training = L.PLANS[plan]
    cfg = getattr(P, preset)
    ops = O.plan_ops(lib, cfg, B, S, dtype, training)
    launches, _ = L.plan_launches(lib, cfg, B, S, dtype, training)
    nl = len(cfg.ch_mult)
    kinds = [o['kind'] for o in ops]
    assert kinds.count(_lib.PLAN_OP_LOGSNR) == 1 and kinds.count(_lib.PLAN_OP_POSE) == 1 and kinds.count(_lib.PLAN_OP_LOSS) == 1
    assert kinds.count(_lib.PLAN_OP_EMB) == nl
    assert kinds.count(_lib.PLAN_OP_RESAMPLE) == 2 * (nl - 1)
    assert kinds.count(_lib.PLAN_OP_CONCAT) == (cfg.num_res_blocks + 1) * nl
    assert kinds.count(_lib.PLAN_OP_ATTN_RESIDUAL) == sum(r['kind'] == _lib.LAUNCH_ATTN for r in launches)
    for o in ops:
        assert (o['B'], o['S'], o['E']) == (B, S, cfg.emb_ch)
        if o['kind'] == _lib.PLAN_OP_EMB:
            # emb_bwd_kernel stores the level's gradient: nothing else may write it
            assert o['acc_x'] == 0 and o['C'] == cfg.emb_ch and o['write_dpe'] == training
        if o['kind'] == _lib.PLAN_OP_POSE:
            assert o['need_grad'] == int(bool(training and (cfg.use_pos_emb or cfg.use_ref_pose_emb)))
            assert (o['pos_emb'], o['ref_pose_emb'], o['ray_convention']) == (cfg.use_pos_emb, cfg.use_ref_pose_emb,
                                                                             _lib.RAYS[cfg.ray_convention])
        if o['kind'] == _lib.PLAN_OP_CONCAT:
            a, b = o['C'], o['C2']
            assert o['copies'] == ((a, a + b, 0, 0, a), (b, a + b, 0, a, b), (a + b, a, 0, 0, a), (a + b, b, a, 0, b))
        if o['kind'] != _lib.PLAN_OP_RESAMPLE:
            continue
        # the backward is the forward's adjoint (RS_DOWN: 0.25 x replicate; RS_UP: the 2x2 sum) times the alias scale
        down = o['rs'] == _lib.RS_DOWN
        assert o['rs'] in (_lib.RS_DOWN, _lib.RS_UP)
        assert (o['fwd_pool'], o['fwd_scale']) == ((1, 0.25) if down else (0, 1.))
        assert o['bwd_pool'] == (0 if down else 1)
        assert o['bwd_scale'] == np.float32(np.float32(0.25 if down else 1.) * np.float32(o['gscale']))
        Ho, Wo = (o['H'] // 2, o['W'] // 2) if down else (2 * o['H'], 2 * o['W'])
        # the alias scale is 1 or the alpha of a residual conv that reads this output at its shape
        assert o['gscale'] == 1. or any(r['kind'] == _lib.LAUNCH_CONV and r['residual'] and r['alpha'] == o['gscale'] and
                                         (r['N'], r['Ho'], r['Wo'], r['Co']) == (o['N'], Ho, Wo, o['C']) for r in launches)
        if not training:
            assert o['gscale'] == 1.
