"""Gradient accumulation, the parts that need no GPU: grad_accum_steps validation, the micro-batch dropout seed scheme and
the k*B batch-shape checks."""
import numpy as np
import pytest

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import train as T


@pytest.mark.parametrize('k', [0, -1, 257, 1.0, 2.5, True, '2', None])
def test_grad_accum_steps_rejects(k):
    with pytest.raises(ValueError):
        T.check_grad_accum_steps(k)
    with pytest.raises(ValueError):
        P.TrainStep(None, grad_accum_steps=k)          # validated before anything touches the state or a device


@pytest.mark.parametrize('k', [1, 2, 4, 256, np.int64(8)])
def test_grad_accum_steps_accepts(k):
    assert T.check_grad_accum_steps(k) == int(k) and type(T.check_grad_accum_steps(k)) is int


def test_micro_batch_seed_scheme():
    assert T.MAX_GRAD_ACCUM_STEPS == 256
    for step in (1, 2, 17, 2 ** 31):
        assert T._micro_batch_seed(step, 0) == T._dropout_seed(step)           # micro-batch 0: the seed without accumulation
    assert T._micro_batch_seed(1, 0) == 1
    assert T._micro_batch_seed(1, 1) == (1 << 32) + 1
    assert T._micro_batch_seed(5, 255) == (255 << 32) + 5
    # distinct over micro-batches and steps, and below the rank bits (40 and up)
    seeds = {T._micro_batch_seed(s, j) for s in (1, 2, 3, 2 ** 32 - 1) for j in range(256)}
    assert len(seeds) == 4 * 256 and max(seeds) < 1 << 40


def _batch(rows, S=4):
    r = np.random.RandomState(0)
    return dict(x=r.rand(rows, S, S, 3), z=r.rand(rows, S, S, 3), logsnr=r.rand(rows), R1=r.rand(rows, 3, 3),
                t1=r.rand(rows, 3), R2=r.rand(rows, 3, 3), t2=r.rand(rows, 3), K=r.rand(rows, 3, 3)), r.rand(rows, S, S, 3)


@pytest.mark.parametrize('k,B', [(1, 2), (2, 2), (4, 3)])
def test_accum_batch_shape_checks(k, B):
    batch, noise = _batch(k * B)
    T.check_accum_batch(batch, noise, None, k, B)
    T.check_accum_batch(batch, noise, np.ones(k * B), k, B)
    with pytest.raises(ValueError, match='cond_mask'):
        T.check_accum_batch(batch, noise, np.ones(B * k + 1), k, B)
    with pytest.raises(ValueError, match='noise'):
        T.check_accum_batch(batch, noise[:-1], None, k, B)
    for key in batch:
        bad = dict(batch)
        bad[key] = batch[key][: (k - 1) * B] if k > 1 else batch[key][:B - 1]
        with pytest.raises(ValueError, match=key):
            T.check_accum_batch(bad, noise, None, k, B)
    with pytest.raises(ValueError):
        T.check_accum_batch(*_batch(B), None, 2 * k, B)        # one micro-batch short of 2k
