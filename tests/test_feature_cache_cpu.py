"""The feature cache (DeepCache) without a GPU: the fp64 cheap forward of tests/feature_cache_ref.py, fed the oracle's own
cached tensor, equals the oracle's full forward exactly; it reads the parameters of the kept blocks and no others; and the
sampler's host-side schedule and argument checks."""
import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.sampling import _check_feature_cache, feature_cache_full_steps
from oracle import xunet_ref as R
from tests import feature_cache_ref as F

SMALL = R.RefConfig(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=2, attn_resolutions=(8, 16, 32), attn_heads=4,
                    dropout=0.1)
THREE = R.RefConfig(ch=32, ch_mult=(1, 2, 2), emb_ch=64, num_res_blocks=1, attn_resolutions=(8,), attn_heads=1,
                    dropout=0.0, use_pos_emb=True, use_ref_pose_emb=True)
FOUR = R.RefConfig(ch=32, ch_mult=(1, 2, 2, 4), emb_ch=32, num_res_blocks=1, attn_resolutions=(4, 8), attn_heads=2,
                   dropout=0.0)
CASES = [(SMALL, 16, lvl) for lvl in (1,)] + [(THREE, 16, lvl) for lvl in (1, 2)] + [(FOUR, 16, lvl) for lvl in (1, 2, 3)]


def _setup(cfg, S, B=2, seed=5):
    params = R.init_params(cfg, S, seed=seed, zero_init=False, bias_std=0.1)
    batch, _ = R.synthetic_batch(B, S, seed=1234)
    cond = torch.tensor([1.0, 0.0][:B], dtype=torch.float64)
    return params, batch, cond


@pytest.mark.parametrize('cfg,S,level', CASES)
def test_shallow_forward_with_oracle_tap_is_the_full_forward(cfg, S, level):
    params, batch, cond = _setup(cfg, S)
    taps = {}
    full = R.xunet_forward(params, batch, cond, cfg, train=False, taps=taps)
    got = F.shallow_forward(params, batch, cond, cfg, level, taps[F.cached_name(cfg, level)])
    assert got.dtype == torch.float64
    assert torch.equal(got, full)


def _groups(params):
    """Parameter groups by top-level block ('ConditioningProcessor_0/<leaf>' for the conditioning's leaves)."""
    out = {}
    for k, v in params.items():
        if k == 'ConditioningProcessor_0':
            out.update({f'{k}/{s}': (k, s) for s in v})
        else:
            out[k] = (k, None)
    return out


def _perturbed(params, where, gen):
    k, s = where
    p = dict(params)
    if s is None:
        p[k] = R.nest({n: t + 0.1 * torch.randn(t.shape, generator=gen, dtype=t.dtype) for n, t in R.flatten(params[k]).items()})
    else:
        sub = dict(params[k])
        node = sub[s]
        sub[s] = (node + 0.1 * torch.randn(node.shape, generator=gen, dtype=node.dtype) if isinstance(node, torch.Tensor) else
                  R.nest({n: t + 0.1 * torch.randn(t.shape, generator=gen, dtype=t.dtype) for n, t in R.flatten(node).items()}))
        p[k] = sub
    return p


@pytest.mark.parametrize('cfg,S,level', [(SMALL, 16, 1), (THREE, 16, 1), (THREE, 16, 2)])
def test_only_kept_blocks_are_read(cfg, S, level):
    params, batch, cond = _setup(cfg, S)
    taps = {}
    R.xunet_forward(params, batch, cond, cfg, train=False, taps=taps)
    deep = taps[F.cached_name(cfg, level)]
    base = F.shallow_forward(params, batch, cond, cfg, level, deep)
    kept = F.kept_blocks(cfg, level)
    groups = _groups(params)
    assert kept <= set(groups) | {'ConditioningProcessor_0/pos_emb', 'ConditioningProcessor_0/ref_pose_emb_first',
                                  'ConditioningProcessor_0/ref_pose_emb_other'}
    gen = torch.Generator().manual_seed(0)
    skipped = []
    for name, where in groups.items():
        out = F.shallow_forward(_perturbed(params, where, gen), batch, cond, cfg, level, deep)
        if name in kept:
            assert not torch.equal(out, base), f'{name} is kept but does not change the output'
        else:
            assert torch.equal(out, base), f'{name} is skipped but changes the output'
            skipped.append(name)
    # what is skipped: every block of the levels >= level, the down ResnetBlock into it and its pose-embedding convs
    n = len(cfg.ch_mult)
    assert f'ResnetBlock_{level - 1}' in skipped and f'XUNetBlock_{n * cfg.num_res_blocks}' in skipped
    assert all(f'ConditioningProcessor_0/Conv_{i}' in skipped for i in range(level, n))


def test_cached_tensor_names():
    # the up ResnetBlocks come after the n - 1 down ones, deepest first
    assert F.cached_name(SMALL, 1) == 'ResnetBlock_1'
    assert [F.cached_name(FOUR, lvl) for lvl in (3, 2, 1)] == ['ResnetBlock_3', 'ResnetBlock_4', 'ResnetBlock_5']
    for bad in (0, 2):
        with pytest.raises(ValueError):
            F.cached_name(SMALL, bad)


@pytest.mark.parametrize('steps,n,expect', [
    (1, 1, [1]), (5, 1, [1, 1, 1, 1, 1]), (7, 3, [1, 0, 0, 1, 0, 0, 1]), (4, 2, [1, 0, 1, 0]), (3, 5, [1, 0, 0]),
    (0, 3, [])])
def test_full_step_pattern(steps, n, expect):
    got = feature_cache_full_steps(steps, n)
    assert got.dtype == bool and got.tolist() == [bool(e) for e in expect]


def test_feature_cache_arguments():
    for n_levels in (2, 3, 4):
        for lvl in range(1, n_levels):
            _check_feature_cache(3, lvl, n_levels)
    _check_feature_cache(1, 1, 1)            # N = 1: every forward full, L unused
    _check_feature_cache(1, 5, 2)
    _check_feature_cache(np.int64(2), np.int32(1), 2)
    for n, lvl, levels in ((0, 1, 2), (-1, 1, 2), (1.5, 1, 2), (True, 1, 2), ('2', 1, 2), (None, 1, 2),
                           (2, 0, 2), (2, 2, 2), (2, 3, 3), (3, 1, 1), (2, 1.0, 2), (1, 0, 2), (2, False, 3)):
        with pytest.raises(ValueError):
            _check_feature_cache(n, lvl, levels)


def test_sampler_rejects_bad_cache_arguments_before_the_gpu():
    model = P.XUNet(ch=32, ch_mult=(1, 2, 2))
    for kw in (dict(cache_interval=0), dict(cache_interval=2, cache_level=3), dict(cache_interval=2, cache_level=0)):
        with pytest.raises(ValueError):
            P.Sampler(model, None, 1, 16, **kw)
