"""Resumable training-state checkpoints: layout of the saved tree (Flax TrainState + optax.adam), round trips, rejection of
foreign trees, and the cond_mask stream gather under a 2-process gloo group.  CPU only: the tree is built and parsed by pure
functions over numpy arrays."""
import os
import socket

import msgpack
import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from novel_view_synthesis_3d_b200 import checkpoint as ck

SPEC = {'Conv_0/kernel': ((1, 3, 3, 3, 4), 0), 'Conv_0/bias': ((4,), 108),
        'GroupNorm_0/GroupNorm_0/scale': ((4,), 112), 'GroupNorm_0/GroupNorm_0/bias': ((4,), 116)}
N = 120


def _bufs(seed):
    r = np.random.RandomState(seed)
    return [r.randn(N).astype(np.float32) for _ in range(4)]      # params, mu, nu, ema


def _tree(seed=0, ema=True, rng=None, add_device_axis=False, step=7):
    p, m, v, e = _bufs(seed)
    t = ck.train_state_tree(ck.leaf_tree(p, SPEC), ck.leaf_tree(m, SPEC), ck.leaf_tree(v, SPEC), count=step, step=step,
                            ema=ck.leaf_tree(e, SPEC) if ema else None, rng=rng, add_device_axis=add_device_axis)
    return t, (p, m, v, e)


def test_layout_known_answer():
    rs = np.random.RandomState(3)
    t, _ = _tree(rng=[ck.rng_state_dict(rs)])
    raw = ck.msgpack_restore(ck.msgpack_serialize(t))
    assert set(raw) == {'step', 'params', 'opt_state', 'ema_params', 'rng'}
    assert set(raw['opt_state']) == {'0', '1'} and raw['opt_state']['1'] == {}
    adam = raw['opt_state']['0']
    assert set(adam) == {'count', 'mu', 'nu'}
    for k in ('step',):
        assert isinstance(raw[k], np.ndarray) and raw[k].shape == () and raw[k].dtype == np.int32 and int(raw[k]) == 7
    assert isinstance(adam['count'], np.ndarray) and adam['count'].shape == () and adam['count'].dtype == np.int32
    assert int(adam['count']) == 7
    for tree in (raw['params'], adam['mu'], adam['nu'], raw['ema_params']):
        assert tree['Conv_0']['kernel'].shape == (1, 3, 3, 3, 4) and tree['Conv_0']['kernel'].dtype == np.float32
        assert tree['GroupNorm_0']['GroupNorm_0']['scale'].shape == (4,)
    assert set(raw['rng']) == {'0'} and raw['rng']['0']['keys'].dtype == np.uint32
    assert raw['rng']['0']['keys'].shape == (624,)
    # ndarray leaves are flax's ExtType(1), the step a 0-d ndarray (not a numpy scalar)
    top = msgpack.unpackb(ck.msgpack_serialize(t), raw=False)
    assert isinstance(top['step'], msgpack.ExtType) and top['step'].code == 1
    assert 'ema_params' not in _tree(ema=False)[0]


@pytest.mark.parametrize('add_device_axis', [False, True])
def test_roundtrip(tmp_path, add_device_axis):
    rs = np.random.RandomState(11)
    rs.random_sample(5)
    mask = np.array([1, 0, 1], np.float32)
    t, (p, m, v, e) = _tree(rng=[ck.rng_state_dict(rs, mask), ck.rng_state_dict(np.random.RandomState(2))],
                            add_device_axis=add_device_axis)
    if add_device_axis:
        assert t['params']['Conv_0']['bias'].shape == (1, 4) and t['step'].shape == (1,)
    path = ck.save_checkpoint(str(tmp_path), t, step=7, prefix='state')
    assert os.path.basename(path) == 'state7'
    r = ck.parse_train_state_tree(ck.msgpack_restore(open(path, 'rb').read()), SPEC, N)
    assert r['step'] == 7 and r['count'] == 7
    for k, ref in (('params', p), ('mu', m), ('nu', v), ('ema', e)):
        assert r[k].dtype == torch.float32 and np.array_equal(r[k].numpy(), ref), k
    assert len(r['rng']) == 2
    fresh = np.random.RandomState(0)
    assert np.array_equal(ck._set_rng_state(fresh, r['rng'][0]), mask)
    assert np.array_equal(fresh.random_sample(8), rs.random_sample(8))
    assert ck._set_rng_state(fresh, r['rng'][1]) is None
    # a state file is still a params checkpoint for the sampler
    params = ck.restore_checkpoint(str(tmp_path), prefix='state')
    assert set(params) == {'Conv_0', 'GroupNorm_0'}
    assert np.array_equal(params['Conv_0']['kernel'].reshape(-1), p[:108])


def test_file_without_ema_parses():
    t, _ = _tree(ema=False)
    r = ck.parse_train_state_tree(ck.msgpack_restore(ck.msgpack_serialize(t)), SPEC, N)
    assert r['ema'] is None and r['rng'] is None


def test_mismatched_leaves_rejected():
    t, _ = _tree()
    bad = dict(t, params=dict(t['params'], Conv_9={'bias': np.zeros(4, np.float32)}))
    with pytest.raises(KeyError, match='parameter tree mismatch'):
        ck.parse_train_state_tree(bad, SPEC, N)
    mu = {'Conv_0': {'kernel': np.zeros((1, 3, 3, 3, 4), np.float32), 'bias': np.zeros(5, np.float32)},
          'GroupNorm_0': t['params']['GroupNorm_0']}
    bad = dict(t, opt_state={'0': dict(t['opt_state']['0'], mu=mu), '1': {}})
    with pytest.raises(ValueError, match='Conv_0/bias'):
        ck.parse_train_state_tree(bad, SPEC, N)


def _state(seed, mask_seed, ema=True, step=0):
    """A TrainState over CPU tensors: save/restore only touch the flat buffers, counters and the mask stream."""
    from novel_view_synthesis_3d_b200.train import TrainState, Adam, AdamState
    from novel_view_synthesis_3d_b200.xunet import ParamTree

    def tree(a):
        t = ParamTree()
        t.flat, t.spec = torch.from_numpy(a.copy()), SPEC
        return t
    p, m, v, e = _bufs(seed)
    return TrainState(step=step, apply_fn=None, params=tree(p), tx=Adam(),
                      opt_state=AdamState(mu=torch.from_numpy(m), nu=torch.from_numpy(v), count=step),
                      ema_params=tree(e) if ema else None, ema_decay=0.999 if ema else None,
                      _mask_rng=np.random.RandomState(mask_seed))


def _worker(rank, world, port, ckpt_dir, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        s = _state(1, 100 + rank, step=5)
        s._mask_rng.random_sample(3)
        ck.save_train_state(ckpt_dir, s, step=5)               # collective: the streams are gathered, rank 0 writes
        fresh = _state(2, 7, step=0)
        ptr = fresh.params.flat.data_ptr()
        assert ck.restore_train_state(ckpt_dir, fresh) is fresh
        assert fresh.params.flat.data_ptr() == ptr               # written in place
        assert torch.equal(fresh.params.flat, s.params.flat) and torch.equal(fresh.ema_params.flat, s.ema_params.flat)
        assert fresh.step == 5 and fresh.opt_state.count == 5
        assert np.array_equal(fresh._mask_rng.random_sample(6), s._mask_rng.random_sample(6))   # this rank's own stream
        out[rank] = 1
    finally:
        dist.destroy_process_group()


def test_gloo_world2_save_restore(tmp_path):
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    out = ctx.Manager().dict()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path), out)) for r in range(2)]
    [p.start() for p in procs]
    [p.join(120) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert dict(out) == {0: 1, 1: 1}
    # restored at another world size: the fresh stream is kept, with a warning
    one = _state(0, 42, ema=False)
    expect = np.random.RandomState(42).random_sample(4)
    with pytest.warns(UserWarning, match='2 ranks'):
        ck.restore_train_state(str(tmp_path), one)
    assert one.step == 5 and np.array_equal(one._mask_rng.random_sample(4), expect)


def test_restore_into_state_with_and_without_ema(tmp_path):
    src = _state(1, 3, ema=False, step=2)
    ck.save_train_state(str(tmp_path), src, step=2)
    dst = _state(2, 4, ema=True)
    ck.restore_train_state(str(tmp_path), dst)
    assert torch.equal(dst.ema_params.flat, src.params.flat)     # no EMA in the file: start it from the params
    src = _state(5, 3, ema=True, step=4)
    ck.save_train_state(str(tmp_path), src, step=4)
    assert sorted(os.listdir(tmp_path)) == ['state4']
    dst = _state(6, 4, ema=False)
    ck.restore_train_state(str(tmp_path), dst)
    assert dst.ema_params is None and torch.equal(dst.opt_state.nu, src.opt_state.nu) and dst.step == 4
    assert ck.restore_train_state(str(tmp_path / 'nope'), dst) is None
