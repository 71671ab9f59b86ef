"""Gradient accumulation over micro-batches in the fused training step: the accumulate backward against the overwriting one
bit for bit on every leaf, TrainStep(grad_accum_steps=k) against k separate forward / backward calls summed in fp32 and one
apply_gradients, graph against eager, the dropout seeds and cond_mask values the micro-batches consume, fp32 parity against
the oracle, and a bit-exact resume."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200 import checkpoint as ck
from novel_view_synthesis_3d_b200.train import _micro_batch_seed
from oracle import xunet_ref as R
from tests.util import np_batch, to_ref_cfg

pytestmark = pytest.mark.gpu

S, B = 64, 2
# tiny 16x16 plan with every optional leaf (pos_emb, ref_pose_emb) and dropout on; the small 64x64 plan is the bench model
TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.1,
            use_pos_emb=True, use_ref_pose_emb=True)
PLANS = {'tiny16': (TINY, 16), 'small64': ({}, 64)}


def _micro(k, seed):
    """k micro-batches of B samples, and the same data as one k*B batch."""
    parts = [R.synthetic_batch(B, S, seed=seed + j) for j in range(k)]
    batch = {key: np.concatenate([np_batch(b)[key] for b, _ in parts]) for key in parts[0][0]}
    noise = np.concatenate([nz.numpy() for _, nz in parts])
    return parts, batch, noise


def _leaf_mismatch(model, s, b, got, want):
    spec = model.param_spec(s, b)
    return [name for name, (shape, off) in spec.items()
            if not torch.equal(got[off:off + int(np.prod(shape))], want[off:off + int(np.prod(shape))])]


# ---- 1. kernel contract ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
@pytest.mark.parametrize('plan', sorted(PLANS))
def test_backward_accumulate_adds_exactly(plan, dtype):
    kw, s = PLANS[plan]
    model = P.XUNet(**kw, dtype=dtype)
    params = P.create_train_state(0, 1, 1e-3, B, s, model=model, zero_init=False).params.flat
    eng = model.engine(B, s, True)
    batch, noise = R.synthetic_batch(B, s, seed=11)
    eng.load_inputs(np_batch(batch), cond_mask=np.array([1.0, 0.0], np.float32), noise=noise.numpy())

    def run(accumulate, g0):
        if g0 is not None:
            eng.grads.copy_(g0)
        eng.forward(params, train=True, seed=1234)
        loss, g = eng.backward(params, accumulate=accumulate)
        torch.cuda.synchronize()
        return float(loss), g.clone()

    loss, g = run(False, None)
    assert bool(torch.isfinite(g).all())
    g0 = torch.randn(g.numel(), generator=torch.Generator().manual_seed(5)).cuda()
    for name in ('ConditioningProcessor_0/Dense_0/kernel', 'ConditioningProcessor_0/Dense_1/bias'):
        shape, off = model.param_spec(s, B)[name]
        assert bool((g[off:off + int(np.prod(shape))] != 0).any()), name    # the log-SNR Dense leaves get a gradient
    loss1, acc = run(True, g0)
    assert loss1 == loss
    bad = _leaf_mismatch(model, s, B, acc, g0 + g)
    assert not bad, bad[:8]
    _, acc0 = run(True, torch.zeros_like(g))
    bad = _leaf_mismatch(model, s, B, acc0, g)
    assert not bad, bad[:8]
    _, again = run(False, g0)                                   # the overwriting backward ignores what the buffer held
    assert torch.equal(again, g)


def test_backward_accumulate_bucket_hook_partitions_the_buffer():
    model = P.XUNet(dtype='bf16')
    params = P.create_train_state(0, 1, 1e-3, B, S, model=model, zero_init=False).params.flat
    eng = model.engine(B, S, True)
    batch, noise = R.synthetic_batch(B, S, seed=12)
    eng.load_inputs(np_batch(batch), cond_mask=np.ones(B, np.float32), noise=noise.numpy())
    ranges = {False: [], True: []}
    for acc in (False, True):
        n = eng.set_bucket_callback(lambda off, cnt, acc=acc: ranges[acc].append((off, cnt)), 1 << 16)
        try:
            eng.forward(params, train=True, seed=3)
            eng.backward(params, accumulate=acc)
        finally:
            eng.set_bucket_callback(None)
        torch.cuda.synchronize()
        assert len(ranges[acc]) == n > 1
    assert ranges[True] == ranges[False]
    end = eng.nparams
    for off, cnt in ranges[True]:                               # descending, contiguous, covering the whole buffer
        assert off + cnt == end
        end = off
    assert end == 0


# ---- 2. TrainStep against k separate forward / backward calls -------------------------------------------------------------
def _new_state(**kw):
    return P.create_train_state(0, 1, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, **kw)


def _manual_update(ref, parts, masks, k):
    """k Engine.forward(seed=s_j) / backward calls, the gradients summed in fp32 in micro-batch order, one apply_gradients
    at grad_scale = 1/k."""
    eng = ref.model.engine(B, S, True)
    acc, losses = None, []
    for j, (b, nz) in enumerate(parts):
        eng.load_inputs(np_batch(b), cond_mask=masks[j], noise=nz.numpy())
        eng.forward(ref.params.flat, train=True, seed=_micro_batch_seed(ref.step + 1, j))
        loss, g = eng.backward(ref.params.flat)
        losses.append(loss.clone())
        acc = g.clone() if acc is None else acc.add_(g)
    ref.grad_scale = 1.0 / k
    ref = ref.apply_gradients(grads=acc)
    ref.grad_scale = 1.0
    return ref, acc, torch.cat(losses)


STATE_KW = {'plain': {}, 'ema': dict(ema_decay=0.9), 'clip+warmup+ema': dict(max_grad_norm=1e-3, warmup_steps=2, ema_decay=0.9)}


@pytest.mark.parametrize('features', sorted(STATE_KW))
@pytest.mark.parametrize('k', [2, 4])
def test_train_step_matches_separate_micro_batches(k, features):
    kw = STATE_KW[features]
    st = _new_state(**kw)
    step = P.TrainStep(st, grad_accum_steps=k)
    ref = _new_state(**kw)
    for i in range(2):
        parts, batch, noise = _micro(k, seed=300 + 10 * i)
        mask = np.random.RandomState(i).randint(0, 2, k * B).astype(np.float32)
        loss = step(batch, noise, cond_mask=mask)
        torch.cuda.synchronize()
        got_loss, got_grads = float(loss), step.eng.grads.clone()
        ref, acc, losses = _manual_update(ref, parts, [mask[j * B:(j + 1) * B] for j in range(k)], k)
        torch.cuda.synchronize()
        assert torch.equal(step.losses, losses), i
        assert got_loss == float(torch.mean(losses, 0, keepdim=True)[0]), i
        assert abs(got_loss - float(losses.double().mean())) <= 1e-6 * abs(got_loss)
        assert torch.equal(got_grads, acc), i
        bufs = [(st.params.flat, ref.params.flat), (st.opt_state.mu, ref.opt_state.mu), (st.opt_state.nu, ref.opt_state.nu)]
        if st.ema_params is not None:
            bufs.append((st.ema_params.flat, ref.ema_params.flat))
        for a, b_ in bufs:
            assert torch.equal(a, b_), i
        if st.clip is not None:
            assert float(st.clip.norm) == float(ref.clip.norm) and float(st.clip.norm) > 1e-3     # clipping active
        assert st.skipped_steps == ref.skipped_steps == 0
    assert step.mode == 'one_graph' and st.step == ref.step == 2 and st.opt_state.count == 2


# ---- 3. graph and eager, repeatability ------------------------------------------------------------------------------------
def _run(k, n_steps, use_graph=True, seed=400, **kw):
    st = _new_state(**kw)
    step = P.TrainStep(st, use_graph=use_graph, grad_accum_steps=k)
    losses = []
    for i in range(n_steps):
        _, batch, noise = _micro(k, seed=seed + 10 * i)
        losses.append(float(step(batch, noise)))          # cond_mask from the host stream
    torch.cuda.synchronize()
    return losses, st, step


def _same_state(a, b):
    return (torch.equal(a.params.flat, b.params.flat) and torch.equal(a.opt_state.mu, b.opt_state.mu) and
            torch.equal(a.opt_state.nu, b.opt_state.nu))


def test_graph_and_eager_agree_and_runs_repeat():
    lg, sg, tg = _run(2, 3)
    le, se, te = _run(2, 3, use_graph=False)
    l2, s2, t2 = _run(2, 3)
    assert tg.mode == 'one_graph' and te.mode == 'eager'
    assert lg == le == l2
    assert _same_state(sg, se) and _same_state(sg, s2)
    assert torch.equal(tg.eng.grads, te.eng.grads) and torch.equal(tg.eng.grads, t2.eng.grads)


# ---- 4. randomness --------------------------------------------------------------------------------------------------------
def test_micro_batches_get_their_own_dropout_seeds_and_masks(lib):
    k = 4
    st = _new_state()
    step = P.TrainStep(st, grad_accum_steps=k)
    for i in range(2):
        _, batch, noise = _micro(k, seed=500 + i)
        step(batch, noise)
        torch.cuda.synchronize()
        want = [_micro_batch_seed(st.step, j) for j in range(k)]
        assert step.seeds.cpu().tolist() == want                 # the seeds the graph replay just used
    assert want[0] == P.train._dropout_seed(st.step)
    n, rate = 1 << 14, st.model.config.dropout
    masks = []
    for sd in want:
        m = torch.empty(n, device='cuda')
        _lib.check(lib.xunet_dropout_mask(m.data_ptr(), n, 0, sd, rate, torch.cuda.current_stream().cuda_stream))
        masks.append(m.cpu())
    for a in range(k):
        for b_ in range(a + 1, k):
            assert not torch.equal(masks[a], masks[b_]), (a, b_)


def test_cond_mask_stream_is_consumed_in_micro_batch_order():
    k = 2
    st = _new_state()
    rng = copy.deepcopy(st._mask_rng)
    step = P.TrainStep(st, grad_accum_steps=k)
    for i in range(3):
        _, batch, noise = _micro(k, seed=600 + i)
        step(batch, noise)
        torch.cuda.synchronize()
        want = np.where(rng.random_sample(k * B) > 0.1, 1, 0).astype(np.float32)
        got = np.concatenate([step.inputs.inp[j]['cond_mask'].cpu().numpy() for j in range(k)])
        assert np.array_equal(got, want), i


def test_k1_runs_the_loop_on_the_engine_buffers():
    """grad_accum_steps=1 is the default step, and its micro-batch loop stages, seeds and scores in the engine's own buffers
    (nothing is allocated twice)."""
    def run(**kw):
        st = _new_state(ema_decay=0.9)
        step = P.TrainStep(st, **kw)
        losses = []
        for i in range(3):
            b, nz = R.synthetic_batch(B, S, seed=700 + i)
            losses.append(float(step(np_batch(b), nz.numpy())))
        torch.cuda.synchronize()
        return losses, st, step

    l0, s0, t0 = run()
    l1, s1, t1 = run(grad_accum_steps=1)
    assert l0 == l1 and _same_state(s0, s1) and torch.equal(s0.ema_params.flat, s1.ema_params.flat)
    assert torch.equal(t0.eng.grads, t1.eng.grads)
    assert t1.inputs is t1.eng.inputs and t1.seeds is t1.eng.seed and t1.loss is t1.eng.loss


def test_wrong_leading_dimension_raises():
    st = _new_state()
    step = P.TrainStep(st, grad_accum_steps=2)
    _, batch, noise = _micro(2, seed=800)
    with pytest.raises(ValueError):
        step({key: v[:B] for key, v in batch.items()}, noise[:B])
    with pytest.raises(ValueError):
        step(batch, noise, cond_mask=np.ones(B, np.float32))
    assert st.step == 0


# ---- 5. fp32 parity against the oracle ------------------------------------------------------------------------------------
def test_accumulation_parity_fp32_against_oracle():
    s, lr, k = 16, 1e-4, 2
    kw = dict(TINY, dropout=0.0)
    model = P.XUNet(**kw, dtype='fp32')
    rcfg = to_ref_cfg(model.config)
    st = P.create_train_state(0, 1, lr, B, s, model=model, zero_init=False)
    step = P.TrainStep(st, grad_accum_steps=k)
    cond = np.array([1.0, 0.0, 0.0, 1.0], np.float32)
    for i in range(2):
        parts = [R.synthetic_batch(B, s, seed=40 + 10 * i + j) for j in range(k)]
        tree = lambda flat: {key: v.double().cpu() for key, v in R.flatten(model.tree_from_flat(flat, s, B)).items()}
        p, m, v = tree(st.params.flat), tree(st.opt_state.mu), tree(st.opt_state.nu)
        gs = [R.loss_and_grads(R.nest(p), b, nz, torch.from_numpy(cond[j * B:(j + 1) * B]).double(), rcfg, train=True)[1]
              for j, (b, nz) in enumerate(parts)]
        g = {key: sum(gj[key] for gj in gs) / k for key in p}
        count = st.opt_state.count
        batch = {key: np.concatenate([np_batch(b)[key] for b, _ in parts]) for key in parts[0][0]}
        step(batch, np.concatenate([nz.numpy() for _, nz in parts]), cond_mask=cond)
        torch.cuda.synchronize()
        got = {key: t.double().cpu() for key, t in R.flatten(st.params).items()}
        for key in p:
            p_new, _, _ = R.adam_update(p[key], g[key], m[key], v[key], count + 1, lr=lr)
            sel = g[key].abs() > 1e-4 * g[key].abs().max() + 1e-12
            if bool(sel.any()):
                assert float((got[key] - p_new)[sel].abs().max()) < 2e-6, (i, key)


# ---- 6. resume ------------------------------------------------------------------------------------------------------------
def test_resume_with_accumulation_is_bit_exact(tmp_path):
    k, kw = 2, dict(ema_decay=0.9, max_grad_norm=1e-3, warmup_steps=3)
    data = [_micro(k, seed=900 + 10 * i)[1:] for i in range(4)]
    ref_losses, ref, _ = _run_on(data, k, kw)
    st = _new_state(**kw)
    step = P.TrainStep(st, grad_accum_steps=k)
    for batch, noise in data[:2]:
        step(batch, noise)
    torch.cuda.synchronize()
    ck.save_train_state(str(tmp_path), st, step=st.step)
    del step, st
    st = P.create_train_state(5, 9, 1e-3, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, **kw)
    assert ck.restore_train_state(str(tmp_path), st) is st and st.step == 2
    step = P.TrainStep(st, grad_accum_steps=k)
    resumed = [float(step(batch, noise)) for batch, noise in data[2:]]
    torch.cuda.synchronize()
    assert resumed == ref_losses[2:]
    assert _same_state(st, ref) and torch.equal(st.ema_params.flat, ref.ema_params.flat)


def _run_on(data, k, kw):
    st = _new_state(**kw)
    step = P.TrainStep(st, grad_accum_steps=k)
    losses = [float(step(batch, noise)) for batch, noise in data]
    torch.cuda.synchronize()
    return losses, st, step


# ---- 7. the example script ------------------------------------------------------------------------------------------------
def test_example_trains_with_accumulation(tmp_path):
    pytest.importorskip('cv2')
    from tests.test_srn_data import _make_tree
    root, ck_dir = str(tmp_path / 'cars'), str(tmp_path / 'ck')
    _make_tree(root, n_inst=2, n_views=4, H=32, W=32)
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(repo, 'examples', 'train_srn.py'), root, '--batch', '2', '--side', '64',
                        '--steps', '3', '--save-every', '2', '--grad-accum-steps', '3', '--ckpt', ck_dir],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert 'training completed' in r.stdout
    raw = ck.msgpack_restore(open(os.path.join(ck_dir, 'state3'), 'rb').read())
    assert int(np.asarray(raw['step']).reshape(-1)[0]) == 3      # one update per 3 micro-batches
