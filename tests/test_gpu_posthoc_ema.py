"""Post-hoc EMA on the GPU: xunet_adam_posthoc_step against a float32 restatement and against xunet_adam_clip_step, the skip
of a non-finite norm, argument errors, the captured TrainStep against an eager run and against a run without averages,
bit-exact resume, and device reconstruction against an fp64 numpy sum."""
import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import checkpoint as ck
from novel_view_synthesis_3d_b200 import posthoc as ph
from oracle import xunet_ref as R
from tests import posthoc_ref as PR
from tests.util import np_batch

pytestmark = pytest.mark.gpu

LR, B1, B2, EPS = 1e-3, 0.9, 0.999, 1e-8
GA, GB = ph.sigma_rel_to_gamma(0.05), ph.sigma_rel_to_gamma(0.10)
CFG = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.1)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _buf(n, offset, fill):
    """n floats on the device starting `offset` floats past a 256-byte aligned allocation."""
    t = torch.empty(n + 4, dtype=torch.float32, device='cuda')[offset: offset + n]
    return t.copy_(fill) if isinstance(fill, torch.Tensor) else t.fill_(fill)


def _posthoc(lib, p, g, m, v, ea, eb, n, step, step_dev, gs, norm=None, max_norm=0.0, warmup=0, skipped=None):
    ptr = lambda t: None if t is None else t.data_ptr()
    return lib.xunet_adam_posthoc_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), ptr(ea), ptr(eb), n, step,
                                       ptr(step_dev), LR, B1, B2, EPS, gs, GA, GB, ptr(norm), max_norm, warmup, ptr(skipped),
                                       _stream())


def _clip(lib, p, g, m, v, n, step, step_dev, gs, norm=None, max_norm=0.0, warmup=0, skipped=None):
    ptr = lambda t: None if t is None else t.data_ptr()
    return lib.xunet_adam_clip_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), None, n, step, ptr(step_dev),
                                    LR, B1, B2, EPS, gs, 0.0, ptr(norm), max_norm, warmup, ptr(skipped), _stream())


# ---- 1. the kernel ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [4 * 2503, 4 * 2503 + 3])
@pytest.mark.parametrize('layout', ['aligned', 'all_offset', 'ema_b_offset'])
@pytest.mark.parametrize('clip', [False, True])
def test_posthoc_kernel_matches_float32_restatement(lib, n, layout, clip):
    g = torch.Generator().manual_seed(11)
    off = 1 if layout == 'all_offset' else 0
    off_b = 0 if layout == 'aligned' else 1      # 'ema_b_offset': only the second average breaks the 16-byte alignment
    p0 = torch.randn(n, generator=g)
    p, m, v = _buf(n, off, p0), _buf(n, off, 0.0), _buf(n, off, 0.0)
    ea, eb = _buf(n, off, torch.randn(n, generator=g)), _buf(n, off_b, torch.randn(n, generator=g))
    pr, mr, vr = p.clone(), m.clone(), v.clone()
    step_dev = torch.zeros(1, dtype=torch.int64, device='cuda')
    norm = torch.zeros(1, device='cuda')
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    a_host, b_host = ea.cpu().numpy(), eb.cpu().numpy()
    # t = 1 overwrites both averages; then small counts, then counts near a million (beta_t close to 1)
    for i, t in enumerate([1, 2, 3, 4, 5, 999_998, 999_999, 1_000_000]):
        gr = _buf(n, off, torch.randn(n, generator=g))
        use_dev = i % 2 == 1
        step_dev.fill_(t)
        sd, sh = (step_dev, 0) if use_dev else (None, t)
        kw = {}
        if clip:
            norm.fill_(0.5 if i % 3 == 0 else 2.0)               # below and above max_norm = 1
            kw = dict(norm=norm, max_norm=1.0, warmup=3, skipped=skipped)
        assert _posthoc(lib, p, gr, m, v, ea, eb, n, sh, sd, 0.5, **kw) == 0, lib.xunet_last_error()
        assert _clip(lib, pr, gr, mr, vr, n, sh, sd, 0.5, **kw) == 0, lib.xunet_last_error()
        torch.cuda.synchronize()
        assert torch.equal(p, pr) and torch.equal(m, mr) and torch.equal(v, vr), t
        pn = pr.cpu().numpy()
        a_host, b_host = PR.f32_update(a_host, pn, t, GA), PR.f32_update(b_host, pn, t, GB)
        if t == 1:
            assert np.array_equal(a_host, pn) and np.array_equal(b_host, pn)
        assert np.array_equal(ea.cpu().numpy(), a_host), t
        assert np.array_equal(eb.cpu().numpy(), b_host), t
    assert int(skipped.item()) == 0


@pytest.mark.parametrize('bad', [float('nan'), float('inf')])
def test_non_finite_norm_touches_neither_average(lib, bad):
    n = 1027
    g = torch.Generator().manual_seed(3)
    p, gr = torch.randn(n, generator=g).cuda(), torch.randn(n, generator=g).cuda()
    m, v = torch.randn(n, generator=g).cuda(), torch.rand(n, generator=g).cuda()
    ea, eb = torch.randn(n, generator=g).cuda(), torch.randn(n, generator=g).cuda()
    before = [t.clone() for t in (p, m, v, ea, eb)]
    norm = torch.full((1,), bad, device='cuda')
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    for t in (1, 7):
        assert _posthoc(lib, p, gr, m, v, ea, eb, n, t, None, 1.0, norm=norm, max_norm=1.0, skipped=skipped) == 0
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip((p, m, v, ea, eb), before))
    assert int(skipped.item()) == 2


def test_posthoc_entry_rejects_bad_arguments(lib):
    n = 64
    p, g, m, v, ea, eb = (torch.zeros(n, device='cuda') for _ in range(6))
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    norm = torch.ones(1, device='cuda')
    ptr = lambda t: None if t is None else t.data_ptr()

    def call(a=ea, b=eb, ga=GA, gb=GB, step=1, norm_=None, max_norm=0.0, warmup=0, sk=None):
        return lib.xunet_adam_posthoc_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), ptr(a), ptr(b), n, step,
                                           None, LR, B1, B2, EPS, 1.0, ga, gb, ptr(norm_), max_norm, warmup, ptr(sk),
                                           _stream())
    assert call() == 0
    for kw in (dict(a=None), dict(b=None), dict(b=ea), dict(ga=-1.0), dict(gb=-3.0), dict(ga=float('nan')),
               dict(gb=float('inf')), dict(step=0), dict(warmup=-1), dict(norm_=norm, max_norm=0.0, sk=skipped),
               dict(norm_=norm, max_norm=1.0, sk=None)):
        assert call(**kw) != 0, kw
        assert lib.xunet_last_error()
    torch.cuda.synchronize()


# ---- 2. the captured training step ---------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def store(tmp_path_factory):
    pytest.importorskip('cv2')
    from tests.test_gpu_device_data import _write_tree
    return P.DeviceScenes(_write_tree(tmp_path_factory.mktemp('srn')), 16)


def _state(posthoc=True, **kw):
    return P.create_train_state(0, 1, 1e-3, 2, 16, model=P.XUNet(**CFG, dtype='bf16'), zero_init=False, max_grad_norm=1.0,
                                posthoc_ema=(0.05, 0.10) if posthoc else None, **kw)


@pytest.mark.parametrize('k', [1, 2])
def test_captured_step_matches_eager_and_leaves_training_unchanged(store, k):
    def run(posthoc, use_graph, steps=4):
        st = _state(posthoc)
        step = P.TrainStep(st, grad_accum_steps=k, data=store, data_seed=5, use_graph=use_graph)
        a0 = None if st.posthoc is None else [f.cpu().numpy() for f in st.posthoc.flats()]
        params, losses = [], []
        for _ in range(steps):
            losses.append(float(step()))
            torch.cuda.synchronize()
            params.append(st.params.flat.cpu().numpy())
        return st, losses, params, a0

    g, lg, pg, a0 = run(True, True)
    e, le, _, _ = run(True, False)
    n, ln, _, _ = run(False, True)
    assert lg == le == ln
    for x, y in ((g, e), (g, n)):
        assert torch.equal(x.params.flat, y.params.flat)
        assert torch.equal(x.opt_state.mu, y.opt_state.mu) and torch.equal(x.opt_state.nu, y.opt_state.nu)
    for fa, fb in zip(g.posthoc.flats(), e.posthoc.flats()):
        assert torch.equal(fa, fb)
    # the graph's warm-up and capture updates left no trace: the averages follow the per-step parameters from count 1
    a, b = a0
    for t, p in enumerate(pg, start=1):
        a, b = PR.f32_update(a, p, t, g.posthoc.gamma[0]), PR.f32_update(b, p, t, g.posthoc.gamma[1])
    assert np.array_equal(g.posthoc.a.flat.cpu().numpy(), a) and np.array_equal(g.posthoc.b.flat.cpu().numpy(), b)


def test_apply_gradients_copy_keeps_the_old_averages():
    S, B = 64, 2
    b, nz = R.synthetic_batch(B, S, seed=3)
    nb = np_batch(b)
    st = P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, posthoc_ema=(0.05, 0.1))
    _, grads = P.apply_model(st, nb['x'], nb['z'], nb['logsnr'], nb['R1'], nb['t1'], nb['R2'], nb['t2'], nb['K'],
                             nz.numpy(), cond_mask=np.ones(B, np.float32))
    old = [f.clone() for f in st.posthoc.flats()]
    new = st.apply_gradients(grads=grads, copy=True)
    torch.cuda.synchronize()
    assert all(torch.equal(f, o) for f, o in zip(st.posthoc.flats(), old))
    assert new.posthoc.a.flat.data_ptr() != st.posthoc.a.flat.data_ptr()
    for f in new.posthoc.flats():                                   # count 1: both averages are the new parameters
        assert torch.equal(f, new.params.flat)


def test_resume_is_bit_exact(store, tmp_path):
    def bufs(st):
        return [t.clone() for t in (st.params.flat, st.opt_state.mu, st.opt_state.nu, *st.posthoc.flats())]

    st = _state()
    step = P.TrainStep(st, data=store, data_seed=9)
    for _ in range(2):
        step()
    ck.save_train_state(str(tmp_path), st, step=st.step)
    del step, st
    ref = _state()
    ref_step = P.TrainStep(ref, data=store, data_seed=9)
    losses = [float(ref_step()) for _ in range(4)]
    torch.cuda.synchronize()
    want = bufs(ref)
    st = _state()
    assert ck.restore_train_state(str(tmp_path), st) is st and st.opt_state.count == 2
    step = P.TrainStep(st, data=store, data_seed=9)
    resumed = [float(step()) for _ in range(2)]
    torch.cuda.synchronize()
    assert resumed == losses[2:]
    assert all(torch.equal(a, b) for a, b in zip(bufs(st), want))
    # averages of other widths, or none at all, are refused
    with pytest.raises(ValueError, match='sigma_rel'):
        ck.restore_train_state(str(tmp_path), P.create_train_state(0, 1, 1e-3, 2, 16, model=P.XUNet(**CFG, dtype='bf16'),
                                                                   posthoc_ema=(0.05, 0.2)))
    plain = _state(posthoc=False)
    ck.save_train_state(str(tmp_path / 'plain'), plain, step=0)
    with pytest.raises(ValueError, match='no post-hoc'):
        ck.restore_train_state(str(tmp_path / 'plain'), _state())


# ---- 3. snapshots and reconstruction on the device ----------------------------------------------------------------------------
def test_device_reconstruct_matches_fp64_numpy(store, tmp_path):
    st = _state()
    step = P.TrainStep(st, data=store, data_seed=2)
    counts = []
    for i in range(6):
        step()
        if (i + 1) % 2 == 0:
            torch.cuda.synchronize()
            ph.save_snapshot(str(tmp_path), st)
            counts.append(st.opt_state.count)
    snaps = ph.load_snapshots(str(tmp_path))
    assert [s.t for s in snaps] == counts
    sr, t = 0.08, 5
    tree = ph.reconstruct(str(tmp_path), sr, t=t)
    c = ph.solve_coefficients([s.t for s in snaps for _ in range(2)], [g for s in snaps for g in s.gamma], t,
                              ph.sigma_rel_to_gamma(sr))
    spec = st.params.spec
    want, mag = np.zeros(st.params.flat.numel()), np.zeros(st.params.flat.numel())
    for i, s in enumerate(snaps):
        a, b = s.averages()
        for ci, tr in ((c[2 * i], a), (c[2 * i + 1], b)):
            x = ci * P.xunet.pack_flat(tr, spec, want.size).double().numpy()
            want += x
            mag += np.abs(x)
    got = P.xunet.pack_flat(tree, spec, want.size).numpy()
    assert got.dtype == np.float32
    # within one fp32 rounding of the fp64 sum, up to the fp64 roundings of the sum itself
    tol = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + 1e-14 * mag
    assert np.all(np.abs(got.astype(np.float64) - want) <= tol)
    # the last count and a tracked width give back the snapshot
    last = P.xunet.pack_flat(ph.reconstruct(str(tmp_path), 0.05), spec, want.size)
    np.testing.assert_allclose(last.numpy(), st.posthoc.a.flat.cpu().numpy(), rtol=1e-5, atol=1e-6)


# ---- 4. the example scripts: train with the averages, rebuild a width, sample it -------------------------------------------
def test_example_scripts_snapshot_rebuild_and_sample(tmp_path):
    pytest.importorskip('cv2')
    import os
    import subprocess
    import sys
    from tests.test_srn_data import _make_tree
    root, ck_dir, out = str(tmp_path / 'cars'), str(tmp_path / 'ck'), str(tmp_path / 'out')
    _make_tree(root, n_inst=2, n_views=4, H=32, W=32)
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def run(script, *args):
        r = subprocess.run([sys.executable, os.path.join(repo, 'examples', script), *args], capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        return r.stdout

    run('train_srn.py', root, '--batch', '2', '--side', '64', '--steps', '3', '--save-every', '2', '--posthoc-ema', '0.05',
        '0.10', '--snapshot-every', '1', '--ckpt', ck_dir)
    assert {'posthoc1', 'posthoc2', 'posthoc3'} <= set(os.listdir(ck_dir))
    run('posthoc_ema_srn.py', '--ckpt', ck_dir, '--sigma-rel', '0.08', '--prefix', 'phema008')
    assert 'phema0083' in os.listdir(ck_dir)
    assert len(ph.load_snapshots(ck_dir)) == 3                     # the rebuilt checkpoint is not taken for a snapshot
    run('sample_srn.py', root, '--ckpt', ck_dir, '--prefix', 'phema008', '--steps', '4', '--side', '64', '--out', out)
    assert os.path.exists(os.path.join(out, 'view_0.png'))
