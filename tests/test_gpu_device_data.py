"""TrainStep(data=DeviceScenes): the batch kernel (xunet_srn_batch) against the host reader and xunet_forward_diffusion, and
training from the device store against the same batches fed through the input slots, bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip('cv2')
import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib, srn_data as D
from novel_view_synthesis_3d_b200.diffusion import min_snr_weights
from novel_view_synthesis_3d_b200.xunet import InputSlots
from tests import device_data_ref as ref

pytestmark = pytest.mark.gpu

CFG = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.1)
NATIVE = 32


def _write_tree(root, counts=(4, 6, 5), side=NATIVE):
    rng = np.random.RandomState(1)
    for i, n in enumerate(counts):
        d = os.path.join(root, f'obj{i:03d}')
        os.makedirs(os.path.join(d, 'rgb'))
        os.makedirs(os.path.join(d, 'pose'))
        with open(os.path.join(d, 'intrinsics.txt'), 'w') as fh:
            fh.write(f'{1.3 * side:.4f} {side / 2:.1f} {side / 2:.1f} 0.\n0. 0. 0.\n1.\n{side} {side}\n')
        for v in range(n):
            cv2.imwrite(os.path.join(d, 'rgb', f'{v:06d}.png'), rng.randint(0, 256, (side, side, 3)).astype(np.uint8))
            q, _ = np.linalg.qr(rng.randn(3, 3))
            pose = np.eye(4)
            pose[:3, :3], pose[:3, 3] = q, rng.randn(3)
            with open(os.path.join(d, 'pose', f'{v:06d}.txt'), 'w') as fh:
                fh.write(' '.join(f'{x:.6f}' for x in pose.reshape(-1)) + '\n')
    return str(root)


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return _write_tree(tmp_path_factory.mktemp('srn'))


def _tables(dev, gamma=None):
    ac = np.cumprod(1. - P.cosine_beta_schedule(1000), axis=0)
    f = lambda a: torch.as_tensor(a, dtype=torch.float32).to(dev)
    return f(np.sqrt(ac)), f(np.sqrt(1. - ac)), None if gamma is None else f(min_snr_weights(gamma))


def _launch(lib, store, slots, slot, count, j, k, rank, world, seed, tabs, p_uncond=0.1, weights=True):
    """One xunet_srn_batch into slot `slot` of `slots`, for the update at Adam count `count`; returns (idx, t) on the host."""
    B = slots.B
    dev = store.device
    step_dev = torch.full((1,), count + 1, dtype=torch.int64, device=dev)
    idx = torch.full((B, 3), -1, dtype=torch.int32, device=dev)
    t = torch.full((B,), -1, dtype=torch.int32, device=dev)
    inp = slots.inp[slot]
    sa, sb, w = tabs
    _lib.check(lib.xunet_srn_batch(C.byref(store.c_store), step_dev.data_ptr(), seed, j, k, rank, world, B, sa.data_ptr(),
                                   sb.data_ptr(), p_uncond, None if w is None else w.data_ptr(), C.byref(slots.cbatch[slot]),
                                   inp['noise'].data_ptr(), inp['loss_weight'].data_ptr() if weights else None,
                                   idx.data_ptr(), t.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), 'srn_batch')
    torch.cuda.synchronize()
    return idx.cpu().numpy().astype(np.int64), t.cpu().numpy()


def _bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a


@pytest.mark.parametrize('S,storage', [(NATIVE, 'uint8'), (16, 'float32')])
def test_batch_kernel_matches_the_host_reader_and_forward_diffusion(tree, lib, S, storage):
    store = D.DeviceScenes(tree, S)
    assert store.storage == storage
    ds = D.SRNScenes(tree, img_sidelength=S)
    B, seed = 5, 0x1234567890ABCDEF
    slots = InputSlots(B, S, 1, store.device)
    eng = P.XUNet(**CFG).engine(B, S, True)
    fd = P.ForwardDiffusion(eng, min_snr_gamma=5.0)
    tabs = _tables(store.device, 5.0)
    for count, j, k, rank, world in ((0, 0, 1, 0, 1), (3, 1, 2, 0, 1), (2, 0, 3, 1, 2), (7, 2, 3, 3, 4), (40, 0, 1, 0, 1)):
        idx, t = _launch(lib, store, slots, 0, count, j, k, rank, world, seed, tabs)
        want = store.draws(count, j, k, rank, world, B, seed=seed)
        assert np.array_equal(idx, want)
        for b in range(B):
            assert tuple(want[b]) == ref.draw(store.first, store.count, store.item_inst, seed, count, j, k, rank, world, B, b)
        inp = slots.inp[0]
        tgt = []
        for b, (i, v, v2) in enumerate(want):
            inst = ds.instances[i]
            assert np.array_equal(_bits(inp['x'][b]), _bits(D.load_rgb(inst['imgs'][v], S)))
            p1, p2 = D.load_pose(inst['poses'][v]), D.load_pose(inst['poses'][v2])
            assert np.array_equal(_bits(inp['R1'][b]), _bits(np.ascontiguousarray(p1[:3, :3])))
            assert np.array_equal(_bits(inp['t1'][b]), _bits(np.ascontiguousarray(p1[:3, 3])))
            assert np.array_equal(_bits(inp['R2'][b]), _bits(np.ascontiguousarray(p2[:3, :3])))
            assert np.array_equal(_bits(inp['t2'][b]), _bits(np.ascontiguousarray(p2[:3, 3])))
            assert np.array_equal(_bits(inp['K'][b]), _bits(inst['K']))
            tgt.append(D.load_rgb(inst['imgs'][v2], S))
        s = D.diffusion_seed(seed, count, j, k, rank)
        assert s == ref.diffusion_seed(seed, count, j, k, rank)
        fd.sample(np.stack(tgt), seed=s)
        torch.cuda.synchronize()
        for key in ('z', 'noise', 'logsnr', 'cond_mask', 'loss_weight'):
            assert np.array_equal(_bits(inp[key]), _bits(eng.inp[key])), key
        assert np.array_equal(t, fd.t.cpu().numpy())


def _state(loss='frobenius', ema=None, B=4, S=16):
    return P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(**CFG), zero_init=False, loss=loss, ema_decay=ema)


def _same_state(a, b):
    for x, y in ((a.params.flat, b.params.flat), (a.opt_state.mu, b.opt_state.mu), (a.opt_state.nu, b.opt_state.nu)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    if a.ema_params is not None:
        assert torch.equal(a.ema_params.flat.view(torch.int32), b.ema_params.flat.view(torch.int32))
    assert a.opt_state.count == b.opt_state.count


@pytest.mark.parametrize('loss,gamma,k', [('frobenius', None, 1), ('mse', 5.0, 1), ('frobenius', None, 2), ('mse', None, 2)])
def test_training_from_the_store_equals_training_on_the_same_batches(tree, lib, loss, gamma, k):
    S, B, seed = 16, 4, 9
    store = D.DeviceScenes(tree, S)
    sa = _state(loss)
    sb = _state(loss)
    step_a = P.TrainStep(sa, data=store, data_seed=seed, grad_accum_steps=k, min_snr_gamma=gamma)
    step_b = P.TrainStep(sb, grad_accum_steps=k)
    slots = InputSlots(B, S, k, store.device)
    tabs = _tables(store.device, gamma)
    for c in range(3):
        for j in range(k):
            _launch(lib, store, slots, j, c, j, k, 0, 1, seed, tabs, weights=loss == 'mse')
        cat = lambda key: torch.cat([slots.inp[j][key] for j in range(k)]).clone()
        batch = {key: cat(key) for key in ('x', 'z', 'logsnr', 'R1', 't1', 'R2', 't2', 'K')}
        la = float(step_a())
        lb = float(step_b(batch, cat('noise'), cond_mask=cat('cond_mask'),
                          loss_weight=cat('loss_weight') if loss == 'mse' else None))
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32), (c, la, lb)
        assert step_a.h2d_bytes == 0
    torch.cuda.synchronize()
    _same_state(sa, sb)


def test_graph_replay_equals_eager(tree):
    store = D.DeviceScenes(tree, 16)
    sa, sb = _state(), _state()
    step_a = P.TrainStep(sa, data=store, data_seed=3)
    step_b = P.TrainStep(sb, data=store, data_seed=3, use_graph=False)
    for _ in range(3):
        la, lb = float(step_a()), float(step_b())
        assert np.float32(la).view(np.int32) == np.float32(lb).view(np.int32)
    assert step_a.mode == 'one_graph' and step_b.mode == 'eager'
    _same_state(sa, sb)


def test_resume_continues_the_data_stream_bit_for_bit(tree, tmp_path):
    store = D.DeviceScenes(tree, 16, cache=str(tmp_path / 'cache'))
    full = _state(ema=0.9)
    step = P.TrainStep(full, data=store, data_seed=5)
    for _ in range(4):
        step()
    part = _state(ema=0.9)
    step = P.TrainStep(part, data=store, data_seed=5)
    for _ in range(2):
        step()
    P.checkpoint.save_train_state(str(tmp_path / 'ckpt'), part, step=part.step)
    store2 = D.DeviceScenes(tree, 16, cache=str(tmp_path / 'cache'))
    assert store2.from_cache
    resumed = _state(ema=0.9)
    assert P.checkpoint.restore_train_state(str(tmp_path / 'ckpt'), resumed) is not None
    step = P.TrainStep(resumed, data=store2, data_seed=5)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    _same_state(full, resumed)


def test_data_step_errors(tree):
    store = D.DeviceScenes(tree, 16)
    st = _state()
    step = P.TrainStep(st, data=store)
    B, S = st.batch_size, st.img_sidelength
    batch = P.create_sample_data(B, S)
    noise = batch.pop('noise')
    with pytest.raises(ValueError):
        step(batch, noise)
    with pytest.raises(ValueError):
        P.TrainStep(P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(**CFG), reference_quirks=True), data=store)
    with pytest.raises(ValueError):
        P.TrainStep(_state(), data=store, min_snr_gamma=5.0)
    with pytest.raises(ValueError):
        P.TrainStep(_state(S=32), data=store)
    other = type('Store', (), dict(S=16, device=torch.device('cuda', 1)))()
    with pytest.raises(ValueError):
        P.TrainStep(_state(), data=other)
    with pytest.raises(ValueError):
        P.TrainStep(_state(), min_snr_gamma=5.0)
    loss = step()
    assert step.h2d_bytes == 0 and np.isfinite(float(loss))
