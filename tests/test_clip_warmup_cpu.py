"""Gradient clipping and learning-rate warm-up without a GPU: known answers of the optax restatements (tests/optax_ref.py),
the four optimizer layouts of the training-state checkpoint, and argument validation."""
import math

import numpy as np
import pytest
import torch

from novel_view_synthesis_3d_b200 import checkpoint as ck
from tests import optax_ref as O

SPEC = {'Conv_0/kernel': ((1, 3, 3, 3, 4), 0), 'Conv_0/bias': ((4,), 108),
        'GroupNorm_0/GroupNorm_0/scale': ((4,), 112), 'GroupNorm_0/GroupNorm_0/bias': ((4,), 116)}
N = 120


# ---- optax restatements ---------------------------------------------------------------------------------------------------
def _grads(scale):
    g = torch.Generator().manual_seed(3)
    return {'a': torch.randn(7, 5, generator=g, dtype=torch.float64) * scale,
            'b': torch.randn(11, generator=g, dtype=torch.float64) * scale}


def _norm(tree):
    return math.sqrt(sum(float((t ** 2).sum()) for t in tree.values()))


def test_clip_by_global_norm_known_answers():
    assert O.clip_by_global_norm([torch.tensor([3.0, 4.0], dtype=torch.float64)], 10.0)[1] == 5.0
    out, n = O.clip_by_global_norm([torch.tensor([3.0, 4.0], dtype=torch.float64)], 1.0)
    assert n == 5.0 and torch.equal(out[0], torch.tensor([0.6, 0.8], dtype=torch.float64))
    small = _grads(0.01)
    out, n = O.clip_by_global_norm(small, 1.0)
    assert n < 1.0 and all(out[k] is small[k] for k in small)           # below the threshold: untouched
    big = _grads(10.0)
    out, n = O.clip_by_global_norm(big, 1.0)
    assert n == pytest.approx(_norm(big), rel=1e-12) and n > 1.0
    assert abs(_norm(out) - 1.0) < 1e-6                                  # above it: rescaled onto the sphere
    for k in big:                                                        # direction kept
        assert torch.allclose(out[k] * n, big[k], rtol=1e-12, atol=0)
    at = {'x': torch.tensor([1.0], dtype=torch.float64)}                 # norm == max_norm: the clip branch (g / n) * c
    out, n = O.clip_by_global_norm(at, 1.0)
    assert n == 1.0 and float(out['x']) == 1.0


def test_warmup_lr_known_answers():
    lr, W = 2e-4, 10
    assert O.warmup_lr(lr, 0, W) == 0.0
    assert O.warmup_lr(lr, W // 2, W) == pytest.approx(lr / 2, rel=1e-15)
    assert O.warmup_lr(lr, W, W) == lr
    assert O.warmup_lr(lr, 2 * W, W) == lr
    assert O.warmup_lr(lr, 0, 0) == lr and O.warmup_lr(lr, 7, 0) == lr


# ---- checkpoint layouts ---------------------------------------------------------------------------------------------------
LAYOUTS = {(False, False), (True, False), (False, True), (True, True)}


def _tree(clip, schedule, skipped=None, add_device_axis=False, count=6):
    r = np.random.RandomState(5)
    p, m, v = (r.randn(N).astype(np.float32) for _ in range(3))
    t = ck.train_state_tree(ck.leaf_tree(p, SPEC), ck.leaf_tree(m, SPEC), ck.leaf_tree(v, SPEC), count=count, step=count,
                            clip=clip, schedule=schedule, skipped=skipped, add_device_axis=add_device_axis)
    return t, (p, m, v)


@pytest.mark.parametrize('clip,schedule', sorted(LAYOUTS))
def test_optimizer_layout_known_answer(clip, schedule):
    t, _ = _tree(clip, schedule, skipped=3 if (clip or schedule) else None)
    raw = ck.msgpack_restore(ck.msgpack_serialize(t))
    opt = raw['opt_state']
    assert set(opt) == {'0', '1'}
    if clip:
        assert opt['0'] == {} and set(opt['1']) == {'0', '1'}
        adam, sched = opt['1']['0'], opt['1']['1']
    else:
        adam, sched = opt['0'], opt['1']
    assert set(adam) == {'count', 'mu', 'nu'} and int(adam['count']) == 6
    if schedule:
        assert set(sched) == {'count'} and sched['count'].dtype == np.int32 and int(sched['count']) == 6
    else:
        assert sched == {}
    if clip or schedule:
        assert raw['skipped_steps'].dtype == np.int64 and int(raw['skipped_steps']) == 3
    else:
        assert 'skipped_steps' not in raw                                # neither feature: exactly the plain layout


@pytest.mark.parametrize('add_device_axis', [False, True])
@pytest.mark.parametrize('clip,schedule', sorted(LAYOUTS))
def test_optimizer_layouts_roundtrip(tmp_path, clip, schedule, add_device_axis):
    skipped = 4 if clip else None
    t, (p, m, v) = _tree(clip, schedule, skipped=skipped, add_device_axis=add_device_axis)
    path = ck.save_checkpoint(str(tmp_path), t, step=6, prefix='state')
    r = ck.parse_train_state_tree(ck.msgpack_restore(open(path, 'rb').read()), SPEC, N)
    assert r['step'] == 6 and r['count'] == 6 and r['skipped'] == (skipped or 0) and r['ema'] is None
    for k, ref in (('params', p), ('mu', m), ('nu', v)):
        assert np.array_equal(r[k].numpy(), ref), k
    params = ck.restore_checkpoint(str(tmp_path), prefix='state')      # still a params checkpoint for the sampler
    assert set(params) == {'Conv_0', 'GroupNorm_0'}
    assert np.array_equal(params['Conv_0']['kernel'].reshape(-1), p[:108])


@pytest.mark.parametrize('clip', [False, True])
def test_mismatched_schedule_count_rejected(clip):
    t, _ = _tree(clip, True)
    sched = t['opt_state']['1']['1'] if clip else t['opt_state']['1']
    sched['count'] = np.asarray(5, dtype=np.int32)
    with pytest.raises(ValueError, match='schedule count'):
        ck.parse_train_state_tree(t, SPEC, N)


def _state(clip, schedule, skipped=0):
    """A TrainState over CPU tensors: save/restore only touch the flat buffers, counters and the mask stream."""
    from novel_view_synthesis_3d_b200.train import TrainState, Adam, AdamState, ClipState
    from novel_view_synthesis_3d_b200.xunet import ParamTree
    r = np.random.RandomState(skipped)
    t = ParamTree()
    t.flat, t.spec = torch.from_numpy(r.randn(N).astype(np.float32)), SPEC
    tx = Adam(max_grad_norm=1.0 if clip else None, warmup_steps=10 if schedule else 0)
    c = None
    if tx.clip_or_warmup:
        c = ClipState(norm=torch.zeros(1), scratch=torch.zeros(4, dtype=torch.float64),
                      skipped=torch.full((1,), skipped, dtype=torch.int64))
    return TrainState(step=3, apply_fn=None, params=t, tx=tx, clip=c,
                      opt_state=AdamState(mu=torch.from_numpy(r.randn(N).astype(np.float32)),
                                          nu=torch.from_numpy(r.rand(N).astype(np.float32)), count=3),
                      _mask_rng=np.random.RandomState(1))


@pytest.mark.parametrize('src', sorted(LAYOUTS))
def test_resume_may_switch_clipping_and_warmup(tmp_path, src):
    """A state saved with any of the four layouts restores into a state with any other."""
    a = _state(*src, skipped=2)
    ck.save_train_state(str(tmp_path), a, step=3)
    for dst in sorted(LAYOUTS):
        b = _state(*dst, skipped=9)
        ck.restore_train_state(str(tmp_path), b)
        assert torch.equal(b.params.flat, a.params.flat) and torch.equal(b.opt_state.nu, a.opt_state.nu)
        assert b.step == 3 and b.opt_state.count == 3
        assert b.skipped_steps == (2 if any(src) and any(dst) else 0), (src, dst)


def test_create_train_state_rejects_bad_settings():
    from novel_view_synthesis_3d_b200 import create_train_state
    for kw in (dict(max_grad_norm=0.0), dict(max_grad_norm=-1.0), dict(max_grad_norm=float('nan')),
               dict(max_grad_norm=float('inf')), dict(warmup_steps=-1), dict(warmup_steps=2.5), dict(warmup_steps=True)):
        with pytest.raises(ValueError):
            create_train_state(0, 1, 1e-3, 2, 16, **kw)
