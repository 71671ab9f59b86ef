"""Host side of the device-resident SRN store (srn_data.DeviceScenes): the draw order, the storage choice and the decode
cache.  CPU only."""
import json
import os

import numpy as np
import pytest

cv2 = pytest.importorskip('cv2')
from novel_view_synthesis_3d_b200 import srn_data as D
from tests import device_data_ref as ref


def _write_tree(root, counts=(3, 5, 4), side=24, ext='png', dtype=np.uint8, seed=0):
    rng = np.random.RandomState(seed)
    for i, n in enumerate(counts):
        d = os.path.join(root, f'obj{i:03d}')
        os.makedirs(os.path.join(d, 'rgb'), exist_ok=True)
        os.makedirs(os.path.join(d, 'pose'), exist_ok=True)
        with open(os.path.join(d, 'intrinsics.txt'), 'w') as fh:
            fh.write(f'{1.1 * side:.4f} {side / 2:.1f} {side / 2:.1f} 0.\n0. 0. 0.\n1.\n{side} {side}\n')
        for v in range(n):
            hi = 65536 if dtype == np.uint16 else 256
            cv2.imwrite(os.path.join(d, 'rgb', f'{v:06d}.{ext}'), rng.randint(0, hi, (side, side + 2, 3)).astype(dtype))
            pose = rng.randn(4, 4)
            with open(os.path.join(d, 'pose', f'{v:06d}.txt'), 'w') as fh:
                fh.write(' '.join(f'{x:.6f}' for x in pose.reshape(-1)) + '\n')
    return str(root)


@pytest.mark.parametrize('n', [1, 2, 3, 7, 64, 1000, 122900])
def test_permutation_is_a_bijection_for_every_epoch(n):
    perms = []
    for seed in (0, 1, 0xDEADBEEFCAFEF00D):
        for epoch in (0, 1, 5):
            p = D.permute(np.arange(n), n, seed, epoch).astype(np.int64)
            assert np.array_equal(np.sort(p), np.arange(n))
            perms.append(p)
    if n >= 7:
        assert all(not np.array_equal(perms[0], q) for q in perms[1:3])      # epochs of one seed differ
    xs = np.unique(np.linspace(0, n - 1, 16).astype(np.int64))
    for seed, epoch in ((0, 0), (3, 2)):
        got = D.permute(xs, n, seed, epoch)
        assert [int(v) for v in got] == [ref.permute(int(x), n, seed, epoch) for x in xs]


def _tables(counts):
    counts = np.asarray(counts, np.int32)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32)
    return first, counts, np.repeat(np.arange(len(counts), dtype=np.int32), counts)


def test_ranks_and_micro_batches_partition_each_update():
    first, counts, inst = _tables([3, 7, 1, 5, 4])
    n = len(inst)
    for c, k, world, B in ((0, 1, 1, 4), (3, 2, 4, 3), (7, 3, 2, 5)):
        draws = []
        for r in range(world):
            for j in range(k):
                d = D.draw_indices(first, counts, inst, 11, c, j, k, r, world, B)
                assert d.shape == (B, 3)
                draws.append(first[d[:, 0]] + d[:, 1])       # source items
                for b in range(B):
                    assert tuple(int(v) for v in d[b]) == ref.draw(first, counts, inst, 11, c, j, k, r, world, B, b)
        # the draws of one update are the draw indices [c k world B, (c+1) k world B): restate them from g directly
        g = np.arange(c * k * world * B, (c + 1) * k * world * B)
        want = np.concatenate([D.permute(g[g // n == e] % n, n, 11, e) for e in np.unique(g // n)]).astype(np.int64)
        assert np.array_equal(np.sort(np.concatenate(draws)), np.sort(want))


def test_every_item_is_a_source_once_per_epoch_and_targets_stay_in_range():
    first, counts, inst = _tables([3, 7, 1, 5, 4])
    n, B = len(inst), 4
    src, v2s = [], []
    for c in range(2 * n // B):
        d = D.draw_indices(first, counts, inst, 5, c, 0, 1, 0, 1, B)
        src.append(first[d[:, 0]] + d[:, 1])
        v2s.append(d)
    src = np.concatenate(src)
    assert np.array_equal(np.sort(src[:n]), np.arange(n)) and np.array_equal(np.sort(src[n:2 * n]), np.arange(n))
    assert not np.array_equal(src[:n], src[n:2 * n])
    d = np.concatenate(v2s)
    assert (d[:, 1] >= 0).all() and (d[:, 1] < counts[d[:, 0]]).all()
    assert (d[:, 2] >= 0).all() and (d[:, 2] < counts[d[:, 0]]).all()
    assert len(np.unique(d[:, 2])) > 1


def test_diffusion_seed_matches_the_restatement():
    for args in ((0, 0, 0, 1, 0), (7, 12, 1, 2, 3), (2 ** 64 - 1, 5, 0, 4, 1)):
        assert D.diffusion_seed(*args) == ref.diffusion_seed(*args)
    assert len({D.diffusion_seed(0, c, j, 2, r) for c in range(3) for j in range(2) for r in range(2)}) == 12


def test_uint8_formula_equals_load_rgb(tmp_path):
    root = _write_tree(tmp_path, side=24)
    for p in sorted(D.glob(os.path.join(root, '*', 'rgb', '*.png'))):
        u = D.load_rgb_u8(p, 24)
        assert u is not None and u.dtype == np.uint8
        a, b = D.u8_to_float(u), D.load_rgb(p, 24)
        assert a.dtype == b.dtype == np.float32 and np.array_equal(a.view(np.int32), b.view(np.int32))
    # every 8-bit value
    u = np.arange(256, dtype=np.uint8)
    assert np.array_equal(D.u8_to_float(u), ((u.astype(np.float32) / 255.0) - 0.5) * 2.0)


@pytest.mark.parametrize('side,S,ext,dtype,storage', [
    (24, 24, 'png', np.uint8, 'uint8'),          # crop is S x S: exact uint8
    (24, 16, 'png', np.uint8, 'float32'),        # resized
    (24, 24, 'png', np.uint16, 'float32'),       # 16-bit
    (24, 24, 'jpg', np.uint8, 'float32'),        # JPEG
])
def test_storage_kind_and_values(tmp_path, side, S, ext, dtype, storage):
    root = _write_tree(tmp_path, side=side, ext=ext, dtype=dtype)
    ds = D.SRNScenes(root, img_sidelength=S)
    a = D.decode_scenes(ds, workers=3)
    assert a['storage'] == storage and str(a['pixels'].dtype) == storage
    assert a['pixels'].shape == (len(ds), S, S, 3)
    assert list(a['count']) == [3, 5, 4] and list(a['first']) == [0, 3, 8] and list(a['item_inst']) == [0] * 3 + [1] * 5 + [2] * 4
    for i, (inst, v) in enumerate(ds.index):
        want = D.load_rgb(ds.instances[inst]['imgs'][v], S)
        got = D.u8_to_float(a['pixels'][i]) if storage == 'uint8' else a['pixels'][i]
        assert np.array_equal(got.view(np.int32), want.view(np.int32))
        pose = D.load_pose(ds.instances[inst]['poses'][v])
        assert np.array_equal(a['R'][i], pose[:3, :3]) and np.array_equal(a['t'][i], pose[:3, 3])
    assert np.array_equal(a['K'][1], ds.instances[1]['K'])


def test_cache_round_trips_and_is_rebuilt_when_the_files_or_S_change(tmp_path):
    root = _write_tree(tmp_path / 'tree', side=24)
    cache = str(tmp_path / 'cache')
    ds = D.SRNScenes(root, img_sidelength=24)
    a, hit = D.load_or_decode(ds, cache)
    assert not hit and json.load(open(os.path.join(cache, 'meta.json')))['storage'] == 'uint8'
    b, hit = D.load_or_decode(D.SRNScenes(root, img_sidelength=24), cache)
    assert hit
    for key in ('pixels', 'R', 't', 'K', 'first', 'count', 'item_inst'):
        assert np.array_equal(a[key], b[key]) and a[key].dtype == b[key].dtype
    # another S: decoded again (float32, resized) and the cache replaced
    c, hit = D.load_or_decode(D.SRNScenes(root, img_sidelength=16), cache)
    assert not hit and c['storage'] == 'float32' and c['pixels'].shape[1] == 16
    _, hit = D.load_or_decode(D.SRNScenes(root, img_sidelength=16), cache)
    assert hit
    # another file list: fewer views per instance
    d, hit = D.load_or_decode(D.SRNScenes(root, img_sidelength=16, max_observations_per_instance=2), cache,
                              max_observations_per_instance=2)
    assert not hit and len(d['item_inst']) == 6
    # an added view
    _write_tree(tmp_path / 'tree', counts=(3, 6, 4), side=24, seed=1)
    e, hit = D.load_or_decode(D.SRNScenes(root, img_sidelength=24), cache)
    assert not hit and len(e['item_inst']) == 13
