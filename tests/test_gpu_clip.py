"""Gradient clipping by global norm and linear learning-rate warm-up in the fused training step: the deterministic norm
kernel against an exact float64 sum, the clip / warm-up Adam kernel against the plain Adam kernel fed the numpy float32
restatement, the non-finite skip, TrainStep against apply_model + apply_gradients, fp32 parity against the oracle, bit-exact
resume, and the example script."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200 import checkpoint as ck
from oracle import xunet_ref as R
from tests import optax_ref as O
from tests.util import np_batch, to_ref_cfg

pytestmark = pytest.mark.gpu

S, B = 64, 2
LR, B1, B2, EPS = 1e-3, 0.9, 0.999, 1e-8


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _buf(n, offset, fill, dtype=torch.float32):
    """n elements on the device starting `offset` elements past a 256-byte aligned allocation."""
    t = torch.empty(n + 4, dtype=dtype, device='cuda')[offset: offset + n]
    return t.copy_(fill) if isinstance(fill, torch.Tensor) else t.fill_(fill)


def _norm(lib, g, gs):
    scratch = torch.full((_lib.GRAD_NORM_SCRATCH,), float('nan'), dtype=torch.float64, device='cuda')
    out = torch.zeros(1, dtype=torch.float32, device='cuda')
    assert lib.xunet_grad_global_norm(g.data_ptr(), g.numel(), gs, scratch.data_ptr(), out.data_ptr(), _stream()) == 0
    torch.cuda.synchronize()
    return out, float(scratch[0])


def _exact_sumsq(g: torch.Tensor, gs: float) -> float:
    x = (g.cpu().numpy() * np.float32(gs)).astype(np.float32).astype(np.float64)   # fp32(g * gs), then exact squares
    return math.fsum(x * x)


# ---- 1. norm kernel -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [4 * 2503 + 3, 5_000_003])
@pytest.mark.parametrize('offset', [0, 1])
@pytest.mark.parametrize('gs', [1.0, 1.0 / 3.0])
def test_global_norm_kernel(lib, n, offset, gs):
    g = _buf(n, offset, torch.randn(n, generator=torch.Generator().manual_seed(n + offset)) * 3.0)
    ref = math.sqrt(_exact_sumsq(g, gs))
    out, sumsq = _norm(lib, g, gs)
    assert abs(math.sqrt(sumsq) - ref) <= 1e-9 * ref, (math.sqrt(sumsq), ref)
    assert float(out) == float(np.float32(math.sqrt(sumsq)))             # the fp64 sum rounded to fp32 once
    out2, sumsq2 = _norm(lib, g, gs)
    assert sumsq2 == sumsq and torch.equal(out, out2)                      # deterministic: same bits every launch


def test_global_norm_kernel_edges(lib):
    z = torch.zeros(8, device='cuda')
    scratch = torch.zeros(_lib.GRAD_NORM_SCRATCH, dtype=torch.float64, device='cuda')
    out = torch.full((1,), 5.0, device='cuda')
    assert lib.xunet_grad_global_norm(z.data_ptr(), 0, 1.0, scratch.data_ptr(), out.data_ptr(), _stream()) == 0
    assert float(out) == 0.0                                               # an empty buffer has norm 0
    for bad in (float('nan'), float('inf')):
        g = torch.ones(1000, device='cuda')
        g[517] = bad
        assert not math.isfinite(float(_norm(lib, g, 1.0)[0]))
    assert lib.xunet_grad_global_norm(None, 8, 1.0, z.data_ptr(), z.data_ptr(), _stream()) != 0
    assert lib.xunet_grad_global_norm(z.data_ptr(), -1, 1.0, z.data_ptr(), z.data_ptr(), _stream()) != 0


# ---- 2. clip / warm-up Adam kernel against the plain Adam kernel ---------------------------------------------------------
class Bufs:
    def __init__(self, n, offset, seed, ema):
        g = torch.Generator().manual_seed(seed)
        self.p = _buf(n, offset, torch.randn(n, generator=g))
        self.m, self.v = _buf(n, offset, 0.0), _buf(n, offset, 0.0)
        self.e = _buf(n, offset, torch.randn(n, generator=g)) if ema else None

    def clone(self):
        c = Bufs.__new__(Bufs)
        c.p, c.m, c.v = self.p.clone(), self.m.clone(), self.v.clone()
        c.e = None if self.e is None else self.e.clone()
        return c

    def all(self):
        return [t for t in (self.p, self.m, self.v, self.e) if t is not None]


def _plain(lib, b: Bufs, g, step, lr, gs, decay=0.99):
    if b.e is None:
        rc = lib.xunet_adam_step(b.p.data_ptr(), g.data_ptr(), b.m.data_ptr(), b.v.data_ptr(), g.numel(), step, None, lr,
                                 B1, B2, EPS, gs, _stream())
    else:
        rc = lib.xunet_adam_ema_step(b.p.data_ptr(), g.data_ptr(), b.m.data_ptr(), b.v.data_ptr(), b.e.data_ptr(), g.numel(),
                                     step, None, lr, B1, B2, EPS, gs, decay, _stream())
    assert rc == 0


def _clip(lib, b: Bufs, g, step, step_dev, gs, norm, max_norm, warmup, skipped, lr=LR, decay=0.99):
    return lib.xunet_adam_clip_step(b.p.data_ptr(), g.data_ptr(), b.m.data_ptr(), b.v.data_ptr(),
                                    None if b.e is None else b.e.data_ptr(), g.numel(), step,
                                    None if step_dev is None else step_dev.data_ptr(), lr, B1, B2, EPS, gs, decay,
                                    None if norm is None else norm.data_ptr(), max_norm, warmup,
                                    None if skipped is None else skipped.data_ptr(), _stream())


def _same(a: Bufs, b: Bufs):
    return all(torch.equal(x, y) for x, y in zip(a.all(), b.all()))


LAYOUTS = [(0, False), (0, True), (1, False), (1, True)]      # (offset, ema)


@pytest.mark.parametrize('offset,ema', LAYOUTS)
def test_clip_kernel_below_threshold_is_plain_adam(lib, offset, ema):
    n, gs = 4 * 2503 + 3, 0.5
    a = Bufs(n, offset, 1, ema)
    b = a.clone()
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    step_dev = torch.zeros(1, dtype=torch.int64, device='cuda')
    gen = torch.Generator().manual_seed(2)
    for step in range(1, 5):
        g = _buf(n, offset, torch.randn(n, generator=gen))
        norm, _ = _norm(lib, g, gs)
        use_dev = step % 2 == 0
        step_dev.fill_(step)
        assert _clip(lib, a, g, 0 if use_dev else step, step_dev if use_dev else None, gs, norm, 1e30, 0, skipped) == 0
        _plain(lib, b, g, step, LR, gs)
        torch.cuda.synchronize()
        assert _same(a, b), step
    assert int(skipped) == 0


@pytest.mark.parametrize('offset,ema', LAYOUTS)
def test_clip_kernel_clipping_matches_float32_restatement(lib, offset, ema):
    n, gs, max_norm = 4 * 2503 + 3, 0.5, 0.75
    a = Bufs(n, offset, 3, ema)
    b = a.clone()
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    gen = torch.Generator().manual_seed(4)
    for step in range(1, 5):
        g = _buf(n, offset, torch.randn(n, generator=gen))
        norm, _ = _norm(lib, g, gs)
        nf = np.float32(float(norm))
        assert nf >= max_norm
        assert _clip(lib, a, g, step, None, gs, norm, max_norm, 0, skipped) == 0
        # optax: (g / norm) * max_norm on the scaled gradient, each operation rounded in float32
        gc = ((g.cpu().numpy() * np.float32(gs)).astype(np.float32) / nf).astype(np.float32) * np.float32(max_norm)
        _plain(lib, b, _buf(n, offset, torch.from_numpy(gc.astype(np.float32))), step, LR, 1.0)
        torch.cuda.synchronize()
        assert _same(a, b), step
    assert int(skipped) == 0


@pytest.mark.parametrize('offset,ema', LAYOUTS)
def test_warmup_kernel_matches_plain_adam_at_lr_t(lib, offset, ema):
    n, gs, W = 4 * 1001 + 2, 1.0, 4
    a = Bufs(n, offset, 5, ema)
    b = a.clone()
    step_dev = torch.zeros(1, dtype=torch.int64, device='cuda')
    gen = torch.Generator().manual_seed(6)
    for step in range(1, 8):
        g = _buf(n, offset, torch.randn(n, generator=gen))
        step_dev.fill_(step)
        assert _clip(lib, a, g, 0, step_dev, gs, None, 0.0, W, None) == 0     # no norm: warm-up only
        _plain(lib, b, g, step, O.warmup_lr(LR, step - 1, W), gs)
        torch.cuda.synchronize()
        assert _same(a, b), step
        if step == 1:
            assert torch.equal(a.p, Bufs(n, offset, 5, ema).p)              # the first update has lr_t = 0


@pytest.mark.parametrize('bad', [float('nan'), float('inf'), float('-inf')])
@pytest.mark.parametrize('ema', [False, True])
def test_non_finite_norm_skips_the_update(lib, bad, ema):
    n, gs = 4 * 777 + 1, 1.0
    a = Bufs(n, 0, 7, ema)
    b = a.clone()
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    gen = torch.Generator().manual_seed(8)
    g1 = _buf(n, 0, torch.randn(n, generator=gen))
    assert _clip(lib, a, g1, 1, None, gs, _norm(lib, g1, gs)[0], 1e30, 0, skipped) == 0
    _plain(lib, b, g1, 1, LR, gs)
    torch.cuda.synchronize()
    before = a.clone()
    g2 = _buf(n, 0, torch.randn(n, generator=gen))
    g2[n // 3] = bad
    norm2 = _norm(lib, g2, gs)[0]
    assert _clip(lib, a, g2, 2, None, gs, norm2, 1e30, 0, skipped) == 0
    torch.cuda.synchronize()
    assert _same(a, before) and int(skipped) == 1                          # nothing touched, the skip counted
    g3 = _buf(n, 0, torch.randn(n, generator=gen))                         # the next finite step proceeds (count 3)
    assert _clip(lib, a, g3, 3, None, gs, _norm(lib, g3, gs)[0], 1e30, 0, skipped) == 0
    _plain(lib, b, g3, 3, LR, gs)
    torch.cuda.synchronize()
    assert _same(a, b) and not _same(a, before) and int(skipped) == 1


def test_clip_kernel_rejects_bad_arguments(lib):
    n = 1027
    a = Bufs(n, 0, 9, True)
    g = _buf(n, 0, 1.0)
    norm = torch.ones(1, device='cuda')
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    ref = a.clone()
    for kw in (dict(max_norm=0.0), dict(max_norm=-1.0), dict(max_norm=float('nan')), dict(warmup=-1),
               dict(skipped=None), dict(decay=1.5), dict(decay=float('nan'))):
        args = dict(norm=norm, max_norm=1.0, warmup=0, skipped=skipped, decay=0.99)
        args.update(kw)
        assert _clip(lib, a, g, 1, None, 1.0, args['norm'], args['max_norm'], args['warmup'], args['skipped'],
                     decay=args['decay']) != 0, kw
        assert lib.xunet_last_error()
    assert lib.xunet_adam_clip_step(None, g.data_ptr(), a.m.data_ptr(), a.v.data_ptr(), None, n, 1, None, LR, B1, B2, EPS,
                                    1.0, 0.0, None, 0.0, 0, None, _stream()) != 0
    torch.cuda.synchronize()
    assert _same(a, ref) and int(skipped) == 0


# ---- 3. TrainStep ---------------------------------------------------------------------------------------------------------
def _batches(n, seed=500):
    return [R.synthetic_batch(B, S, seed=seed + i) for i in range(n)]


def _new_state(**kw):
    return P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, **kw)


def test_inactive_clipping_does_not_perturb_training():
    batches = _batches(3)
    cond = np.array([1.0, 0.0], dtype=np.float32)

    def run(**kw):
        st = _new_state(**kw)
        step = P.TrainStep(st)
        losses, norms = [], []
        for b, nz in batches:
            losses.append(float(step(np_batch(b), nz.numpy(), cond_mask=cond)))
            norms.append(None if step.grad_norm is None else float(step.grad_norm))
        torch.cuda.synchronize()
        return losses, norms, st

    l0, n0, s0 = run()
    l1, n1, s1 = run(max_grad_norm=1e30, warmup_steps=0)
    assert l0 == l1, (l0, l1)
    assert torch.equal(s0.params.flat, s1.params.flat)
    assert torch.equal(s0.opt_state.mu, s1.opt_state.mu) and torch.equal(s0.opt_state.nu, s1.opt_state.nu)
    assert n0 == [None] * 3 and all(math.isfinite(x) and x > 0 for x in n1)
    assert s1.skipped_steps == 0 and s0.skipped_steps == 0


def test_train_step_matches_apply_model_and_apply_gradients():
    batches = _batches(3, seed=600)
    cond = np.array([1.0, 0.0], dtype=np.float32)
    kw = dict(max_grad_norm=1e-3, warmup_steps=2, ema_decay=0.9)

    st = _new_state(**kw)
    step = P.TrainStep(st)
    losses, norms = [], []
    for b, nz in batches:
        losses.append(float(step(np_batch(b), nz.numpy(), cond_mask=cond)))
        norms.append(float(step.grad_norm))
        # grad_norm is the norm of the averaged gradient the engine just produced
        ref = float(torch.linalg.vector_norm(step.eng.grads.double()))
        assert abs(norms[-1] - ref) <= 1e-6 * ref
    torch.cuda.synchronize()
    assert step.mode == 'one_graph' and all(x > 1e-3 for x in norms)        # clipping active on every step

    ref = _new_state(**kw)
    ref_losses, ref_norms = [], []
    for b, nz in batches:
        nb = np_batch(b)
        loss, grads = P.apply_model(ref, nb['x'], nb['z'], nb['logsnr'], nb['R1'], nb['t1'], nb['R2'], nb['t2'], nb['K'],
                                    nz.numpy(), cond_mask=cond)
        ref = P.update_model(ref, grads)
        ref_losses.append(float(loss))
        ref_norms.append(float(ref.clip.norm))
    torch.cuda.synchronize()
    assert losses == ref_losses, (losses, ref_losses)
    assert norms == ref_norms, (norms, ref_norms)
    for a, b_ in ((st.params.flat, ref.params.flat), (st.opt_state.mu, ref.opt_state.mu),
                  (st.opt_state.nu, ref.opt_state.nu), (st.ema_params.flat, ref.ema_params.flat)):
        assert torch.equal(a, b_)
    assert st.step == ref.step == 3 and st.skipped_steps == ref.skipped_steps == 0


@pytest.mark.parametrize('use_graph', [True, False])
def test_train_step_skips_a_non_finite_step(use_graph):
    (b0, nz0), (b1, nz1) = _batches(2, seed=650)
    cond = np.ones(B, np.float32)
    st = _new_state(max_grad_norm=1.0, ema_decay=0.9)
    step = P.TrainStep(st, use_graph=use_graph)
    before = [t.clone() for t in (st.params.flat, st.opt_state.mu, st.opt_state.nu, st.ema_params.flat)]
    bad = nz0.numpy().copy()
    bad[0, 3, 5, 1] = np.inf                       # loss = inf; its gradient (eps - inf) / inf = NaN reaches the leaves
    loss = float(step(np_batch(b0), bad, cond_mask=cond))     # also the first call: warm-up and capture run on it
    torch.cuda.synchronize()
    assert not math.isfinite(loss) and not math.isfinite(float(step.grad_norm))
    assert st.skipped_steps == 1 and st.step == 1 and st.opt_state.count == 1
    for a, b_ in zip((st.params.flat, st.opt_state.mu, st.opt_state.nu, st.ema_params.flat), before):
        assert torch.equal(a, b_)
    loss = float(step(np_batch(b1), nz1.numpy(), cond_mask=cond))
    torch.cuda.synchronize()
    assert math.isfinite(loss) and st.skipped_steps == 1 and st.step == 2
    assert not torch.equal(st.params.flat, before[0]) and bool(torch.isfinite(st.params.flat).all())


# ---- 4. fp32 parity against the oracle ------------------------------------------------------------------------------------
TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.0)


def test_clip_warmup_parity_fp32_against_oracle():
    s, b, lr, W = 16, 2, 1e-4, 2
    model = P.XUNet(**TINY, dtype='fp32')
    rcfg = to_ref_cfg(model.config)
    batches = [R.synthetic_batch(b, s, seed=40 + i) for i in range(3)]
    cond = np.array([1.0, 0.0])

    def ref_step(st, batch, noise):
        tree = lambda flat: {k: v.double().cpu() for k, v in R.flatten(model.tree_from_flat(flat, s, b)).items()}
        p, m, v = tree(st.params.flat), tree(st.opt_state.mu), tree(st.opt_state.nu)
        _, g, _ = R.loss_and_grads(R.nest(p), batch, noise, torch.from_numpy(cond), rcfg, train=True)
        return p, m, v, g

    # max_norm: a fifth of the first step's norm, so clipping is active on every step with a wide margin
    probe = P.create_train_state(0, 1, lr, b, s, model=model, zero_init=False)
    max_norm = 0.2 * O.clip_by_global_norm(ref_step(probe, *batches[0])[3], 1e30)[1]
    st = P.create_train_state(0, 1, lr, b, s, model=model, zero_init=False, max_grad_norm=max_norm, warmup_steps=W)
    for i, (batch, noise) in enumerate(batches):
        p, m, v, g = ref_step(st, batch, noise)
        g_clip, n_ref = O.clip_by_global_norm(g, max_norm)
        count = st.opt_state.count
        nb = np_batch(batch)
        _, grads = P.apply_model(st, nb['x'], nb['z'], nb['logsnr'], nb['R1'], nb['t1'], nb['R2'], nb['t2'], nb['K'],
                                 noise.numpy(), cond_mask=cond)
        st = P.update_model(st, grads)
        norm = float(st.clip.norm)
        assert abs(norm - n_ref) <= 2e-4 * n_ref, (i, norm, n_ref)
        assert (norm >= max_norm) == (n_ref >= max_norm) and n_ref >= 1.05 * max_norm, i
        lr_t = O.warmup_lr(lr, count, W)
        got = {k: t.double().cpu() for k, t in R.flatten(st.params).items()}
        for k in p:
            p_new, _, _ = R.adam_update(p[k], g_clip[k], m[k], v[k], count + 1, lr=lr_t)
            sel = g[k].abs() > 1e-4 * g[k].abs().max() + 1e-12
            if bool(sel.any()):
                assert float((got[k] - p_new)[sel].abs().max()) < 2e-6, (i, k)
    assert st.skipped_steps == 0


# ---- 5. resume ------------------------------------------------------------------------------------------------------------
def _state_bufs(st):
    return [t.clone() for t in (st.params.flat, st.opt_state.mu, st.opt_state.nu, st.ema_params.flat)]


def test_resume_with_clipping_and_warmup_is_bit_exact(tmp_path):
    batches = _batches(5, seed=800)
    nan_steps = (1, 4)                              # skipped updates: one before the save, one after

    def feed(step, i):
        b, nz = batches[i]
        nz = nz.numpy().copy()
        if i in nan_steps:
            nz[0, 0, 0, 0] = np.inf                # a non-finite gradient, as in test_train_step_skips_a_non_finite_step
        return float(step(np_batch(b), nz))        # cond_mask from the host stream

    kw = dict(max_grad_norm=1e-3, warmup_steps=3, ema_decay=0.9)
    st = _new_state(**kw)
    step = P.TrainStep(st)
    for i in range(2):
        feed(step, i)
    assert st.skipped_steps == 1
    ck.save_train_state(str(tmp_path), st, step=st.step)
    del step, st

    ref = _new_state(**kw)
    ref_step = P.TrainStep(ref)
    losses = [feed(ref_step, i) for i in range(5)]
    torch.cuda.synchronize()
    want = _state_bufs(ref)
    assert ref.skipped_steps == 2

    st = P.create_train_state(5, 9, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, **kw)
    assert ck.restore_train_state(str(tmp_path), st) is st and st.step == 2 and st.skipped_steps == 1
    step = P.TrainStep(st)
    resumed = [feed(step, i) for i in range(2, 5)]
    torch.cuda.synchronize()
    assert np.array_equal(resumed, losses[2:], equal_nan=True), (resumed, losses)
    for a, b_ in zip(_state_bufs(st), want):
        assert torch.equal(a, b_)
    assert st.skipped_steps == 2

    ck.restore_train_state(str(tmp_path), ref)     # in place, into the already captured TrainStep
    assert ref.skipped_steps == 1
    again = [feed(ref_step, i) for i in range(2, 5)]
    torch.cuda.synchronize()
    assert np.array_equal(again, losses[2:], equal_nan=True), (again, losses)
    for a, b_ in zip(_state_bufs(ref), want):
        assert torch.equal(a, b_)
    assert ref.skipped_steps == 2


# ---- 6. the example script ------------------------------------------------------------------------------------------------
def test_example_trains_with_clipping_and_warmup_and_resumes(tmp_path):
    pytest.importorskip('cv2')
    from tests.test_srn_data import _make_tree
    root, ck_dir = str(tmp_path / 'cars'), str(tmp_path / 'ck')
    _make_tree(root, n_inst=2, n_views=4, H=32, W=32)
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def run(*args):
        r = subprocess.run([sys.executable, os.path.join(repo, 'examples', 'train_srn.py'), root, *args],
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        return r.stdout

    common = ['--batch', '2', '--side', '64', '--save-every', '2', '--ema-decay', '0.99', '--max-grad-norm', '1',
              '--warmup-steps', '2', '--ckpt', ck_dir]
    log = run(*common, '--steps', '3')
    assert 'grad norm' in log and 'skipped steps (non-finite gradient norm): 0' in log, log
    raw = ck.msgpack_restore(open(os.path.join(ck_dir, 'state3'), 'rb').read())
    assert raw['opt_state']['0'] == {} and int(raw['opt_state']['1']['1']['count']) == 3
    log = run(*common, '--steps', '5', '--resume')
    assert 'resumed from step 3' in log and 'training completed' in log
    assert sorted(os.listdir(ck_dir)) == ['ema4', 'model4', 'state5']
