"""Weight EMA fused into the Adam kernel, and resumable training state: the kernel against a float32 restatement, EMA on /
off giving the same training bits, copy semantics, bit-exact resume through save_train_state / restore_train_state, and
sampling from the EMA weights."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import checkpoint as ck
from oracle import xunet_ref as R
from tests.util import np_batch

pytestmark = pytest.mark.gpu

S, B = 64, 2
DECAY = 0.9


def _stream():
    return torch.cuda.current_stream().cuda_stream


def ema_ref(ema: np.ndarray, p_new: np.ndarray, decay: float) -> np.ndarray:
    """float32 restatement of the kernel: d and 1-d formed in double then rounded, each product and the sum rounded."""
    d, omd = np.float32(decay), np.float32(1.0 - decay)
    return (d * ema.astype(np.float32) + omd * p_new.astype(np.float32)).astype(np.float32)


def _buf(n, offset, fill):
    """n floats on the device starting `offset` floats past a 256-byte aligned allocation."""
    t = torch.empty(n + 4, dtype=torch.float32, device='cuda')[offset: offset + n]
    return t.copy_(fill) if isinstance(fill, torch.Tensor) else t.fill_(fill)


# ---- 1. kernel ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('layout', ['aligned', 'all_offset', 'ema_offset'])
def test_fused_adam_ema_kernel(lib, layout):
    n = 4 * 2503 + 3                              # float4 main loop + ragged scalar tail
    g = torch.Generator().manual_seed(7)
    off = 0 if layout == 'aligned' else 1
    off_e = 1 if layout != 'aligned' else 0       # 'ema_offset': only the EMA buffer breaks the 16-byte alignment
    p0, e0 = torch.randn(n, generator=g), torch.randn(n, generator=g)
    p, m, v = _buf(n, off, p0), _buf(n, off, 0.0), _buf(n, off, 0.0)
    ema = _buf(n, off_e, e0)
    pr, mr, vr = p.clone(), m.clone(), v.clone()
    step_dev = torch.zeros(1, dtype=torch.int64, device='cuda')
    e_host = e0.numpy()
    for step in range(1, 6):
        gr = _buf(n, off, torch.randn(n, generator=g))
        use_dev = step % 2 == 0                   # alternate host step and device step counter
        step_dev.fill_(step)
        sd, sh = (step_dev.data_ptr(), 0) if use_dev else (None, step)
        assert lib.xunet_adam_ema_step(p.data_ptr(), gr.data_ptr(), m.data_ptr(), v.data_ptr(), ema.data_ptr(), n, sh, sd,
                                       1e-3, 0.9, 0.999, 1e-8, 0.5, 0.99, _stream()) == 0
        assert lib.xunet_adam_step(pr.data_ptr(), gr.data_ptr(), mr.data_ptr(), vr.data_ptr(), n, sh, sd, 1e-3, 0.9, 0.999,
                                   1e-8, 0.5, _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(p, pr) and torch.equal(m, mr) and torch.equal(v, vr), step
        e_host = ema_ref(e_host, pr.cpu().numpy(), 0.99)
        assert np.array_equal(ema.cpu().numpy(), e_host), step


def test_fused_adam_ema_decay_limits_and_bad_arguments(lib):
    n = 1027
    g = torch.Generator().manual_seed(1)
    p, gr = torch.randn(n, generator=g).cuda(), torch.randn(n, generator=g).cuda()
    m, v = torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    ema = torch.randn(n, generator=g).cuda()
    args = lambda e, d: (p.data_ptr(), gr.data_ptr(), m.data_ptr(), v.data_ptr(), e, n, 1, None, 1e-3, 0.9, 0.999, 1e-8,
                         1.0, d, _stream())
    assert lib.xunet_adam_ema_step(*args(ema.data_ptr(), 0.0)) == 0
    torch.cuda.synchronize()
    assert torch.equal(ema, p)                    # decay 0: the EMA is the current weights
    e1 = ema.clone() + 1.0
    ema.copy_(e1)
    assert lib.xunet_adam_ema_step(*args(ema.data_ptr(), 1.0)) == 0
    torch.cuda.synchronize()
    assert torch.equal(ema, e1)                   # decay 1: the EMA never moves
    for e, d in ((None, 0.999), (ema.data_ptr(), -0.1), (ema.data_ptr(), 1.5), (ema.data_ptr(), float('nan'))):
        assert lib.xunet_adam_ema_step(*args(e, d)) != 0
        assert lib.xunet_last_error()
    assert torch.equal(ema, e1)


# ---- 2./3. training with EMA ----------------------------------------------------------------------------------------------
def _batches(n, seed=500):
    return [R.synthetic_batch(B, S, seed=seed + i) for i in range(n)]


def test_ema_does_not_perturb_training():
    batches = _batches(3)
    cond = np.array([1.0, 0.0], dtype=np.float32)

    def run(ema_decay):
        st = P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, ema_decay=ema_decay)
        step = P.TrainStep(st)
        e0 = None if st.ema_params is None else st.ema_params.flat.cpu().numpy()
        losses, snaps = [], []
        for b, nz in batches:
            losses.append(float(step(np_batch(b), nz.numpy(), cond_mask=cond)))
            torch.cuda.synchronize()
            snaps.append((st.params.flat.cpu().numpy(), None if st.ema_params is None else st.ema_params.flat.cpu().numpy()))
        return losses, st, snaps, e0

    l0, s0, _, _ = run(None)
    l1, s1, snaps, e = run(DECAY)
    assert l0 == l1, (l0, l1)
    assert torch.equal(s0.params.flat, s1.params.flat)
    assert torch.equal(s0.opt_state.mu, s1.opt_state.mu) and torch.equal(s0.opt_state.nu, s1.opt_state.nu)
    assert not np.array_equal(e, snaps[0][0])                    # the weights moved
    for i, (p, ema) in enumerate(snaps):                         # the graph's warm-up / capture updates left no trace
        e = ema_ref(e, p, DECAY)
        assert np.array_equal(ema, e), i


def test_apply_gradients_copy_keeps_the_old_ema():
    b, nz = R.synthetic_batch(B, S, seed=3)
    nb = np_batch(b)
    st = P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, ema_decay=DECAY)
    _, grads = P.apply_model(st, nb['x'], nb['z'], nb['logsnr'], nb['R1'], nb['t1'], nb['R2'], nb['t2'], nb['K'],
                             nz.numpy(), cond_mask=np.ones(B, np.float32))
    e_old, p_old = st.ema_params.flat.clone(), st.params.flat.clone()
    new = st.apply_gradients(grads=grads, copy=True)
    torch.cuda.synchronize()
    assert torch.equal(st.ema_params.flat, e_old) and torch.equal(st.params.flat, p_old)
    assert new.ema_params.flat.data_ptr() != st.ema_params.flat.data_ptr()
    assert not torch.equal(new.params.flat, p_old)
    assert np.array_equal(new.ema_params.flat.cpu().numpy(), ema_ref(e_old.cpu().numpy(), new.params.flat.cpu().numpy(), DECAY))
    assert new.ema_decay == DECAY and new.opt_state.count == 1


def test_create_train_state_rejects_bad_decay():
    for d in (-0.5, 1.01):
        with pytest.raises(ValueError):
            P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), ema_decay=d)


# ---- 4. resume ------------------------------------------------------------------------------------------------------------
def _state_bufs(st):
    return [t.clone() for t in (st.params.flat, st.opt_state.mu, st.opt_state.nu, st.ema_params.flat)]


def test_resume_is_bit_exact(tmp_path):
    batches = _batches(4, seed=700)
    feed = lambda step, i: float(step(np_batch(batches[i][0]), batches[i][1].numpy()))     # cond_mask from the host stream

    # 2 steps, save
    st = P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, ema_decay=DECAY)
    step = P.TrainStep(st)
    for i in range(2):
        feed(step, i)
    ck.save_train_state(str(tmp_path), st, step=st.step)
    del step, st

    # the uninterrupted run
    ref = P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, ema_decay=DECAY)
    ref_step = P.TrainStep(ref)
    losses = [feed(ref_step, i) for i in range(4)]
    torch.cuda.synchronize()
    want = _state_bufs(ref)

    # a fresh state (other init, other mask stream) restored from the step-2 file, new TrainStep
    st = P.create_train_state(5, 9, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, ema_decay=DECAY)
    assert ck.restore_train_state(str(tmp_path), st) is st and st.step == 2 and st.opt_state.count == 2
    step = P.TrainStep(st)
    resumed = [feed(step, i) for i in range(2, 4)]
    torch.cuda.synchronize()
    assert resumed == losses[2:], (resumed, losses)
    for a, b_ in zip(_state_bufs(st), want):
        assert torch.equal(a, b_)

    # the same file restored in place into the already captured TrainStep of the uninterrupted run
    ptrs = [t.data_ptr() for t in (ref.params.flat, ref.opt_state.mu, ref.opt_state.nu, ref.ema_params.flat)]
    ck.restore_train_state(str(tmp_path), ref)
    assert ptrs == [t.data_ptr() for t in (ref.params.flat, ref.opt_state.mu, ref.opt_state.nu, ref.ema_params.flat)]
    again = [feed(ref_step, i) for i in range(2, 4)]
    torch.cuda.synchronize()
    assert again == losses[2:], (again, losses)
    for a, b_ in zip(_state_bufs(ref), want):
        assert torch.equal(a, b_)


# ---- 5. sampling the EMA weights --------------------------------------------------------------------------------------------
def test_sampler_on_ema_weights_and_ema_checkpoint(tmp_path):
    st = P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, ema_decay=DECAY)
    step = P.TrainStep(st)
    for b, nz in _batches(2, seed=900):
        step(np_batch(b), nz.numpy(), cond_mask=np.ones(B, np.float32))
    torch.cuda.synchronize()
    assert not torch.equal(st.ema_params.flat, st.params.flat)
    ck.save_checkpoint(str(tmp_path), st.ema_params, step=2, prefix='ema', add_device_axis=True)
    tree = ck.restore_checkpoint(str(tmp_path), prefix='ema')
    batch = np_batch(R.synthetic_batch(B, S, seed=11)[0])
    a = P.Sampler(P.XUNet(dtype='bf16'), st.ema_params, B, S, steps=4, w=3.0).sample(batch, seed=2)
    b = P.Sampler(P.XUNet(dtype='bf16'), tree, B, S, steps=4, w=3.0).sample(batch, seed=2)
    assert torch.equal(a, b)


# ---- the example scripts: train with EMA, resume, sample the EMA ----------------------------------------------------------
def test_example_scripts_train_resume_and_sample_ema(tmp_path):
    pytest.importorskip('cv2')
    from tests.test_srn_data import _make_tree
    root, ck_dir, out = str(tmp_path / 'cars'), str(tmp_path / 'ck'), str(tmp_path / 'out')
    _make_tree(root, n_inst=2, n_views=4, H=32, W=32)
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def run(script, *args):
        r = subprocess.run([sys.executable, os.path.join(repo, 'examples', script), root, *args], capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        return r.stdout

    common = ['--batch', '2', '--side', '64', '--save-every', '2', '--ema-decay', '0.99', '--ckpt', ck_dir]
    run('train_srn.py', *common, '--steps', '3')
    assert sorted(os.listdir(ck_dir)) == ['ema2', 'model2', 'state3']
    assert ck.restore_checkpoint(ck_dir, prefix='state')['Conv_0']['kernel'].shape == (1, 3, 3, 3, 32)
    log = run('train_srn.py', *common, '--steps', '5', '--resume')
    assert 'resumed from step 3' in log
    assert sorted(os.listdir(ck_dir)) == ['ema4', 'model4', 'state5']
    run('sample_srn.py', '--ckpt', ck_dir, '--prefix', 'ema', '--steps', '4', '--side', '64', '--out', out)
    assert os.path.exists(os.path.join(out, 'view_0.png'))
