"""The mean-squared epsilon loss (create_train_state(loss='mse')) on the GPU: fp32 parity of the loss and every gradient leaf
against the fp64 reference, the output-gradient seed bit for bit against a float32 numpy restatement, the global-batch
property under gradient accumulation, determinism and exact scaling in the weights, the unchanged Frobenius default,
ForwardDiffusion's min-SNR-gamma weights, and graph replay against eager."""
import math

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.diffusion import min_snr_weights
from oracle import xunet_ref as R
from tests import mse_ref
from tests.util import np_batch, to_ref_cfg

pytestmark = pytest.mark.gpu

TINY = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=1, attn_resolutions=(8, 16), attn_heads=2, dropout=0.0)
SMALL = dict(ch=32, ch_mult=(1, 2), emb_ch=32, num_res_blocks=2, attn_resolutions=(8, 16, 32), attn_heads=4, dropout=0.0)


def _weights(n, seed):
    return np.random.RandomState(seed).uniform(0.1, 3.0, n).astype(np.float32)


def _batch(n, s, seed):
    batch, noise = R.synthetic_batch(n, s, seed=seed)
    return np_batch(batch), noise.numpy()


def _apply(state, batch, noise, cond, w=None):
    loss, grads = P.apply_model(state, batch['x'], batch['z'], batch['logsnr'], batch['R1'], batch['t1'], batch['R2'],
                                batch['t2'], batch['K'], noise, cond_mask=cond, loss_weight=w)
    torch.cuda.synchronize()
    return float(loss), grads.flat.clone()


# ---- 1. fp32 verify mode against the fp64 reference ------------------------------------------------------------------------
@pytest.mark.parametrize('weighted', [False, True])
def test_fp32_loss_and_gradients_match_the_reference(weighted):
    S, B = 64, 2
    model = P.XUNet(**SMALL, dtype='fp32')
    rcfg = to_ref_cfg(model.config)
    ref_params = R.init_params(rcfg, S, seed=7, zero_init=False, bias_std=0.1)
    state = P.create_train_state(0, 1, 1e-4, B, S, model=model, loss='mse')
    state.params.flat.copy_(model.flat_from_tree(ref_params, S, B))
    batch, noise = R.synthetic_batch(B, S, seed=1234)
    cond = np.array([1.0, 0.0])
    w = _weights(B, 3) if weighted else None
    loss_ref, grads_ref, _ = mse_ref.loss_and_grads(ref_params, batch, noise, torch.from_numpy(cond), rcfg, loss='mse',
                                                    loss_weight=None if w is None else torch.from_numpy(w).double())
    loss, g = _apply(state, np_batch(batch), noise.numpy(), cond, w)
    assert abs(loss - float(loss_ref)) / float(loss_ref) <= 1e-3
    gflat = R.flatten(model.tree_from_flat(g, S, B))
    total_ref = math.sqrt(sum(float((x ** 2).sum()) for x in grads_ref.values()))
    bad = {}
    for key, gr in grads_ref.items():
        err = float(torch.linalg.norm((gflat[key].double().cpu() - gr).reshape(-1)))
        # per-leaf relative error, floored as in the Frobenius parity test so leaves with negligible gradient do not dominate
        rel = err / (float(torch.linalg.norm(gr.reshape(-1))) + 1e-3 * total_ref / math.sqrt(len(grads_ref)))
        if rel > 2e-3:
            bad[key] = rel
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]


# ---- 2. the output-gradient seed, bit for bit ---------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['bf16', 'fp32'])
def test_output_gradient_seed_is_bit_exact(dtype):
    S, B = 16, 3
    model = P.XUNet(**TINY, dtype=dtype)
    state = P.create_train_state(0, 1, 1e-4, B, S, model=model, zero_init=False, loss='mse')
    eng = model.engine(B, S, True)
    batch, noise = _batch(B, S, 21)
    w = _weights(B, 4)
    w[1] = 0.0                                                        # a removed sample: its seed is exactly zero
    eng.load_inputs(batch, cond_mask=np.array([1.0, 0.0, 1.0], np.float32), noise=noise, loss_weight=w)
    eps = eng.forward(state.params.flat, train=True, seed=5).cpu().numpy()
    loss, _ = eng.backward(state.params.flat, loss='mse', loss_weight=eng.inp['loss_weight'])
    torch.cuda.synchronize()
    per = S * S * 3
    r = (eps - noise.astype(np.float32)).reshape(B, per)                  # float32 subtraction, rounded once
    c = np.array([np.float32(2.0 * np.float64(wb) / (B * per)) for wb in w], np.float32)
    seed = (c[:, None] * r).astype(np.float32)                            # float32 product, rounded once
    want = torch.from_numpy(seed)
    if dtype == 'bf16':
        want = want.to(torch.bfloat16).float()
    got = eng.read_tap('out_both_frames', grad=True).cpu().reshape(B, 2, per)
    assert torch.equal(got[:, 0], torch.zeros(B, per))
    assert torch.equal(got[:, 1].view(torch.int32), want.view(torch.int32))
    want_loss = float(np.sum(w.astype(np.float64) * np.sum(r.astype(np.float64) ** 2, axis=1)) / (B * per))
    assert abs(float(loss) - want_loss) <= np.spacing(np.float32(want_loss))


# ---- 3. the global-batch property ---------------------------------------------------------------------------------------------
def _accumulated_and_whole(loss, weighted):
    """Summed gradient / 2 and mean loss of TrainStep(grad_accum_steps=2) on two B-sample micro-batches, and the gradient and
    loss of apply_model on the same 2B samples as one batch, from the same parameters (fp32, dropout 0)."""
    S, B, k = 16, 2, 2
    model = P.XUNet(**TINY, dtype='fp32')
    st_k = P.create_train_state(0, 1, 1e-4, B, S, model=model, zero_init=False, loss=loss)
    st_1 = P.create_train_state(0, 1, 1e-4, k * B, S, model=model, zero_init=False, loss=loss)
    st_1.params.flat.copy_(st_k.params.flat)
    batch, noise = _batch(k * B, S, 31)
    cond = np.array([1.0, 0.0, 1.0, 1.0], np.float32)
    w = _weights(k * B, 5) if weighted else None
    whole_loss, whole = _apply(st_1, batch, noise, cond, w)
    step = P.TrainStep(st_k, grad_accum_steps=k)
    acc_loss = float(step(batch, noise, cond_mask=cond, loss_weight=w))
    torch.cuda.synchronize()
    return model, acc_loss, step.eng.grads.clone() / k, whole_loss, whole, (S, B)


# Besides the key biases (a key bias shifts every score of a query by the same amount, which the softmax ignores), the TINY
# 16² plan has conv biases whose every path to the loss enters a 32-channel GroupNorm of 32 groups: one channel per group, so
# a constant shift of a channel is normalised away
ZERO_GRAD_TINY16 = {'XUNetBlock_0/ResnetBlock_0/Conv_0/bias', 'XUNetBlock_5/ResnetBlock_0/Conv_0/bias',
                    'XUNetBlock_6/ResnetBlock_0/Conv_0/bias', 'XUNetBlock_6/ResnetBlock_0/Conv_1/bias'}


@pytest.mark.parametrize('weighted', [False, True])
def test_accumulated_mse_gradient_is_the_gradient_of_the_whole_batch(weighted):
    model, acc_loss, acc, whole_loss, whole, (S, B) = _accumulated_and_whole('mse', weighted)
    assert acc_loss == pytest.approx(whole_loss, rel=1e-6)
    top = float(whole.abs().max())
    bad = []
    for name, (shape, off) in model.param_spec(S, B).items():
        a, b = acc[off:off + int(np.prod(shape))], whole[off:off + int(np.prod(shape))]
        if name.endswith('AttnLayer_0/DenseGeneral_1/bias') or name in ZERO_GRAD_TINY16:
            # leaves whose true gradient is exactly zero: what both sides hold is rounding, held to an absolute bound
            ok = float((a - b).abs().max()) <= 1e-5 * top
        else:
            ok = float(torch.linalg.norm(a - b)) <= 1e-5 * float(torch.linalg.norm(b))
        if not ok:
            bad.append(name)
    assert not bad, bad[:8]


def test_accumulated_frobenius_gradient_is_not_the_gradient_of_the_whole_batch():
    """Why the MSE loss exists: with the Frobenius norm each micro-batch's gradient r/||r|| has unit scale whatever the
    error, so accumulating two micro-batches is not one batch of twice the size."""
    _, acc_loss, acc, whole_loss, whole, _ = _accumulated_and_whole('frobenius', False)
    assert abs(acc_loss - whole_loss) / whole_loss > 1e-2
    assert float(torch.linalg.norm(acc - whole)) > 1e-2 * float(torch.linalg.norm(whole))


# ---- 4. determinism and exact scaling ----------------------------------------------------------------------------------------
def test_mse_steps_repeat_bit_for_bit_and_scale_exactly_with_the_weights():
    S, B = 64, 2
    batch, noise = _batch(B, S, 41)
    cond = np.array([1.0, 0.0], np.float32)
    w = _weights(B, 6)

    def run(weights):
        st = P.create_train_state(0, 1, 1e-4, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, loss='mse')
        loss, g = _apply(st, batch, noise, cond, weights)
        st = P.update_model(st, st.model.tree_from_flat(g, S, B))
        torch.cuda.synchronize()
        return loss, g, st.params.flat.clone()

    l1, g1, p1 = run(w)
    l2, g2, p2 = run(w)
    assert l1 == l2 and torch.equal(g1, g2) and torch.equal(p1, p2)
    l3, g3, _ = run(2 * w)
    assert bool((g1 != 0).any())
    assert torch.equal(g3, 2 * g1)                         # a power-of-two scale of every seed commutes with each rounding
    assert l3 == 2 * l1


# ---- 5. the default is unchanged ------------------------------------------------------------------------------------------------
def test_explicit_frobenius_is_the_default_bit_for_bit():
    S, B = 64, 2

    def run(**kw):
        st = P.create_train_state(0, 1, 1e-4, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, **kw)
        step = P.TrainStep(st)
        losses = [float(step(*_batch(B, S, 50 + i))) for i in range(2)]
        torch.cuda.synchronize()
        return losses, st, step

    l0, s0, t0 = run()
    l1, s1, t1 = run(loss='frobenius')
    assert s0.loss == s1.loss == 'frobenius'
    assert l0 == l1 and torch.equal(s0.params.flat, s1.params.flat) and torch.equal(t0.eng.grads, t1.eng.grads)
    assert torch.equal(s0.opt_state.mu, s1.opt_state.mu) and torch.equal(s0.opt_state.nu, s1.opt_state.nu)


def test_weights_on_a_frobenius_state_are_rejected():
    S, B = 16, 2
    st = P.create_train_state(0, 1, 1e-4, B, S, model=P.XUNet(**TINY), zero_init=False)
    batch, noise = _batch(B, S, 60)
    with pytest.raises(ValueError):
        P.TrainStep(st)(batch, noise, loss_weight=np.ones(B, np.float32))
    with pytest.raises(ValueError):
        _apply(st, batch, noise, np.ones(B, np.float32), np.ones(B, np.float32))
    eng = st.model.engine(B, S, True)
    with pytest.raises(ValueError):
        eng.backward(st.params.flat, loss_weight=eng.inp['loss_weight'])
    with pytest.raises(ValueError):
        eng.backward(st.params.flat, loss='l2')
    assert st.step == 0


# ---- 6. ForwardDiffusion with min-SNR-gamma ------------------------------------------------------------------------------------
def test_forward_diffusion_fills_the_min_snr_weights_of_the_device_timesteps():
    S, B, gamma = 16, 8, 5.0
    eng = P.XUNet(**TINY).engine(B, S, True)
    fd = P.ForwardDiffusion(eng, min_snr_gamma=gamma)
    assert fd.loss_weight is not None and fd.loss_weight.data_ptr() == eng.inp['loss_weight'].data_ptr()
    table = min_snr_weights(gamma).astype(np.float32)
    x0 = np.random.RandomState(0).uniform(-1, 1, (B, S, S, 3)).astype(np.float32)
    for seed in (1, 2):
        fd.sample(x0, seed)
        torch.cuda.synchronize()
        t = fd.t.cpu().numpy()
        assert np.array_equal(fd.loss_weight.cpu().numpy(), table[t])
    t_fixed = np.array([0, 1, 10, 100, 500, 900, 998, 999], np.int32)
    fd.sample(x0, 3, t=t_fixed)
    torch.cuda.synchronize()
    assert np.array_equal(fd.loss_weight.cpu().numpy(), table[t_fixed])
    assert P.ForwardDiffusion(eng).loss_weight is None


# ---- 7. graph replay against eager ----------------------------------------------------------------------------------------------
def test_graph_step_with_staged_weights_equals_the_eager_step():
    S, B, k = 64, 2, 2
    data = [_batch(k * B, S, 70 + i) for i in range(3)]
    weights = [_weights(k * B, 8), _weights(k * B, 9), None]

    def run(use_graph, last_weights):
        st = P.create_train_state(0, 1, 1e-4, B, S, model=P.XUNet(dtype='bf16'), zero_init=False, loss='mse',
                                  max_grad_norm=1.0)
        step = P.TrainStep(st, use_graph=use_graph, grad_accum_steps=k)
        losses = [float(step(batch, noise, loss_weight=w))
                  for (batch, noise), w in zip(data, weights[:2] + [last_weights])]
        torch.cuda.synchronize()
        return losses, st, step

    lg, sg, tg = run(True, None)                            # no weights after weighted steps: all 1 again
    le, se, te = run(False, np.ones(k * B, np.float32))
    assert tg.mode == 'one_graph' and te.mode == 'eager'
    assert lg == le
    assert torch.equal(sg.params.flat, se.params.flat) and torch.equal(tg.eng.grads, te.eng.grads)
    assert torch.equal(sg.opt_state.mu, se.opt_state.mu) and torch.equal(sg.opt_state.nu, se.opt_state.nu)
