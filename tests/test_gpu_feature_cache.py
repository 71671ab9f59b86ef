"""The feature cache (DeepCache, `xunet_set_feature_cache`) on the GPU: a cheap forward right after a full one on the same
inputs gives the full forward's bits; the cached tensor survives cheap forwards; a cheap forward matches the fp64 cheap
forward of tests/feature_cache_ref.py fed the oracle's cached tensor; it launches exactly the kernels of the kept ops;
the Sampler's default is unchanged and its cached chains are reproducible; and the argument errors."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import xunet_ref as R
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200.xunet import Engine
import novel_view_synthesis_3d_b200 as P
from tests import feature_cache_ref as F
from tests.test_gpu_model import FOUR, SMALL, THREE, FWD_TOL, _pool_from_batch, _setup
from tests.util import np_batch, rel_l2

pytestmark = pytest.mark.gpu

THREE_POS = dict(THREE, use_pos_emb=True, use_ref_pose_emb=True)
# (config, side, batch): the small 64^2 model and two configs of three and four levels
CONFIGS = [(SMALL, 64, 2), (THREE_POS, 32, 2), (FOUR, 64, 1)]
CASES = [(c, S, B, lvl) for c, S, B in CONFIGS for lvl in range(1, len(c['ch_mult']))]
IDS = [f"L{len(c['ch_mult'])}-S{S}-level{lvl}" for c, S, B, lvl in CASES]


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def _set(lib, eng, level):
    assert lib.xunet_set_feature_cache(eng.h, level) == 0, lib.xunet_last_error()


def _batch(B, S, seed):
    batch, _ = R.synthetic_batch(B, S, seed=seed)
    return batch


def _run(lib, eng, flat, batch, cond, level):
    _set(lib, eng, level)
    try:
        eng.load_inputs(np_batch(batch), cond_mask=cond.numpy())
        out = eng.forward(flat, train=False).clone()
    finally:
        _set(lib, eng, 0)
    torch.cuda.synchronize()
    return out


def _engine(cfgd, S, B, dtype):
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, dtype)
    eng = model.engine(B, S, False)
    flat = model.flat_from_tree(ref_params, S, B)
    cond = torch.tensor(([1.0, 0.0] * B)[:B], dtype=torch.float64)
    return model, rcfg, ref_params, eng, flat, batch, cond


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
@pytest.mark.parametrize('cfgd,S,B,level', CASES, ids=IDS)
def test_cheap_after_full_on_the_same_inputs_is_bit_identical(lib, cfgd, S, B, level, dtype):
    """Checks the skip set, the statistics that survive (the concat norm reads the cached tensor's sums) and the FiLM branch."""
    model, rcfg, ref_params, eng, flat, batch, cond = _engine(cfgd, S, B, dtype)
    full = _run(lib, eng, flat, batch, cond, 0)
    cheap = _run(lib, eng, flat, batch, cond, level)
    assert torch.equal(cheap, full)
    assert bool(torch.isfinite(full).all())


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
@pytest.mark.parametrize('cfgd,S,B,level', CASES, ids=IDS)
def test_cache_survives_cheap_forwards_and_matches_the_oracle(lib, cfgd, S, B, level, dtype):
    model, rcfg, ref_params, eng, flat, a, cond = _engine(cfgd, S, B, dtype)
    b, b2 = _batch(B, S, 77), _batch(B, S, 91)
    name = F.cached_name(rcfg, level)
    full_a = _run(lib, eng, flat, a, cond, 0)
    deep = eng.read_tap(name)
    cheap_b = _run(lib, eng, flat, b, cond, level)
    last = _run(lib, eng, flat, b2, cond, level)
    assert torch.equal(eng.read_tap(name), deep)
    _run(lib, eng, flat, a, cond, 0)
    assert torch.equal(_run(lib, eng, flat, b2, cond, level), last)
    assert not torch.equal(cheap_b, full_a) and not torch.equal(last, cheap_b)
    # parity: the fp64 cheap forward on B, fed the oracle's cached tensor at A
    taps = {}
    R.xunet_forward(ref_params, a, cond, rcfg, train=False, taps=taps)
    ref = F.shallow_forward(ref_params, b, cond, rcfg, level, taps[name])
    t = taps[name]
    assert rel_l2(deep, t.reshape(-1, *t.shape[-3:])) < 2 * FWD_TOL[dtype]
    assert rel_l2(cheap_b, ref) < FWD_TOL[dtype]


def _leaf_names(eng):
    return list(eng.spec)


def _block(leaf):
    parts = leaf.split('/')
    return '/'.join(parts[:2]) if parts[0] == 'ConditioningProcessor_0' else parts[0]


def _skipped_kernels(lib, eng, rcfg, level):
    """The kernels the plan's skipped ops launch in a full forward: one per conv and attention launch and, for an output a
    norm reads, the fold of its fp64 channel sums, after a statistics kernel when the launch has no statistics epilogue; one
    per GroupNorm, residual-path resample (the resampling ResnetBlocks) and log-SNR FiLM embedding; two channel copies per
    concat (the up XUNetBlocks)."""
    kept = F.kept_blocks(rcfg, level)
    names = _leaf_names(eng)
    n = 0
    owner = None
    info = _lib.XunetLaunchInfo()
    for i in range(lib.xunet_plan_launch_count(eng.h)):
        assert lib.xunet_plan_launch(eng.h, i, C.byref(info)) == 0
        if info.kind == _lib.LAUNCH_CONV:
            leaf = names[info.leaf]
            owner = _block(leaf)
            # outputs some norm reads: the input conv, a ResnetBlock's Conv_0 and Conv_1 (its output)
            normed = leaf == 'Conv_0/kernel' or (owner != 'Conv_1' and leaf.endswith(('/Conv_0/kernel', '/Conv_1/kernel'))
                                                 and not owner.startswith('ConditioningProcessor_0'))
        else:
            normed = True                     # the attention block's output, read by the next norm
        if owner not in kept:
            n += 1 + (normed and 1 + (not info.emits_stats))
    _, _, _, up, _ = F._names(rcfg)
    up_blocks = {b for lvl in up for b in lvl}
    blocks = {_block(x) for x in names}
    for b in blocks - kept:
        n += sum(x.startswith(b + '/') and x.endswith('/scale') for x in names)
        n += b.startswith('ResnetBlock_')
        n += 2 * (b in up_blocks)
        n += b.startswith('ConditioningProcessor_0/Conv_')       # the level's OP_EMB
    return n


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
@pytest.mark.parametrize('cfgd,S,B,level', CASES, ids=IDS)
def test_cheap_forward_launches_the_kept_ops_only(lib, cfgd, S, B, level, dtype):
    model, rcfg, ref_params, eng, flat, batch, cond = _engine(cfgd, S, B, dtype)
    eng.load_inputs(np_batch(batch), cond_mask=cond.numpy())
    full, _ = eng.count_kernels(flat)
    _set(lib, eng, level)
    try:
        cheap, _ = eng.count_kernels(flat)
    finally:
        _set(lib, eng, 0)
    assert eng.count_kernels(flat)[0] == full
    assert cheap < full
    assert full - cheap == _skipped_kernels(lib, eng, rcfg, level)


SAMPLERS = [('ddpm', 3.0), ('ddim', 3.0), ('dpmpp_2m', 3.0), ('ddpm', None), ('dpmpp_2m', None)]


def _sample(model, tree, B, S, nb, **kw):
    samp = P.Sampler(model, tree, B, S, steps=kw.pop('steps', 7), **kw)
    views, poses, K, tp = _pool_from_batch(nb)
    tp = {k: np.concatenate([tp[k], poses[k]], 1) for k in ('R', 't')}      # two targets: the second one's pool has two views
    z = samp.sample(nb, seed=3)
    zv, ch = samp.sample_views(views, poses, K, tp, seed=3, return_choices=True)
    return z, zv, ch


@pytest.mark.parametrize('method,w', SAMPLERS)
def test_default_sampler_is_unchanged(method, w):
    cfgd, S, B = THREE_POS, 32, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, 'bf16')
    nb = np_batch(batch)
    before = _sample(model, tree, B, S, nb, w=w, method=method)
    cached = _sample(model, tree, B, S, nb, w=w, method=method, cache_interval=3, cache_level=2)   # on the same engine
    explicit = _sample(model, tree, B, S, nb, w=w, method=method, cache_interval=1, cache_level=1)
    after = _sample(model, tree, B, S, nb, w=w, method=method)
    for got in (explicit, after):
        assert torch.equal(got[0], before[0]) and torch.equal(got[1], before[1])
        assert (got[2] == before[2]).all()
    assert not torch.equal(cached[0], before[0])


@pytest.mark.parametrize('method,w,dyn', [('ddpm', 3.0, None), ('ddim', None, None), ('dpmpp_2m', 3.0, 0.995)])
@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
def test_cached_sampler_is_reproducible(method, w, dyn, dtype):
    cfgd, S, B = SMALL, 64, 2
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, dtype)
    nb = np_batch(batch)
    kw = dict(w=w, method=method, dynamic_threshold=dyn, steps=8)
    graph = _sample(model, tree, B, S, nb, cache_interval=3, cache_level=1, **kw)
    eager = _sample(model, tree, B, S, nb, cache_interval=3, cache_level=1, use_graph=False, **kw)
    again = _sample(model, tree, B, S, nb, cache_interval=3, cache_level=1, **kw)
    for got in (eager, again):
        assert torch.equal(got[0], graph[0]) and torch.equal(got[1], graph[1]) and (got[2] == graph[2]).all()
    assert bool(torch.isfinite(graph[0]).all()) and bool(torch.isfinite(graph[1]).all())
    # a view is drawn on full steps only (positions 0, 3, 6, ...); the cheap ones hold it
    ch = graph[2]
    assert ch.shape[0] == 2 and ch.shape[1] >= 4
    for k in range(ch.shape[1]):
        assert (ch[:, k] == ch[:, k - k % 3]).all()
    # the first step is a full one: it equals the uncached sampler's first step
    first = {}
    for n in (1, 3):
        samp = P.Sampler(model, tree, B, S, cache_interval=n, cache_level=1, **kw)
        first[n] = samp.sample(nb, seed=3, _max_steps=1)
    assert torch.equal(first[1], first[3])
    assert not torch.equal(_sample(model, tree, B, S, nb, **kw)[0], graph[0])


def test_argument_errors(lib):
    cfgd, S, B = FOUR, 64, 1
    model, rcfg, ref_params, tree, batch, _ = _setup(cfgd, S, B, 'bf16')
    train_eng = model.engine(B, S, True)
    assert lib.xunet_set_feature_cache(train_eng.h, 1) != 0
    assert b'training' in lib.xunet_last_error()
    eng = Engine(model.config, B, S, False)          # a fresh handle: no forward yet
    for bad in (-1, 4, 9):
        assert lib.xunet_set_feature_cache(eng.h, bad) != 0
        assert b'outside' in lib.xunet_last_error()
    flat = model.flat_from_tree(ref_params, S, B)
    eng.load_inputs(np_batch(batch), cond_mask=np.ones(B, np.float32))
    _set(lib, eng, 2)
    with pytest.raises(RuntimeError, match='needs a full forward'):
        eng.forward(flat, train=False)
    _set(lib, eng, 0)
    eng.forward(flat, train=False)
    _set(lib, eng, 3)
    eng.forward(flat, train=False)
    _set(lib, eng, 3)
    eng.forward(flat, train=False)                   # the level-3 tensor is still the full forward's
    _set(lib, eng, 1)                                # but the cheap forwards at 3 recomputed the level-1 tensor
    with pytest.raises(RuntimeError, match='needs a full forward'):
        eng.forward(flat, train=False)
    _set(lib, eng, 0)
    eng.forward(flat, train=False)
    _set(lib, eng, 1)
    eng.forward(flat, train=False)
    _set(lib, eng, 0)
    torch.cuda.synchronize()
    assert lib.xunet_set_feature_cache(None, 0) != 0
