"""v-prediction without a GPU: the v tables of `sampler_table` against an fp64 restatement, an oracle denoiser through the
step formula (exact predictions recover x0; a perturbation of v reaches x0 scaled by sigma_t, one of eps by sqrt(1/abar - 1)),
`v_target` and the v min-SNR weights against their formulas, argument validation, and `prediction` in the training-state
checkpoint."""
import numpy as np
import pytest
import torch

from novel_view_synthesis_3d_b200 import checkpoint as ck
from novel_view_synthesis_3d_b200 import create_train_state
from novel_view_synthesis_3d_b200.diffusion import diffusion_tables, min_snr_weights, v_target
from novel_view_synthesis_3d_b200.sampling import METHODS, PREDICTIONS, Schedule, sampler_table
from tests import solver_ref as S
from tests.test_train_state_checkpoint import N, SPEC, _state

C_RECIP, C_RECIPM1 = 0, 1
CASES = [('ddpm', 0.0, 1000, 'linear'), ('ddpm', 0.0, 25, 'linear'), ('ddim', 0.0, 50, 'linear'), ('ddim', 0.5, 25, 'logsnr'),
         ('dpmpp_2m', 0.0, 25, 'logsnr')]


@pytest.mark.parametrize('method,eta,steps,spacing', CASES)
def test_v_table_matches_an_fp64_restatement(method, eta, steps, spacing):
    """Columns 0 and 1 are sqrt(abar) and sqrt(1 - abar) of each row's timestep; every other column is the eps table's."""
    sched = Schedule(steps, spacing=spacing)
    for lag in (True, False):
        eps, f_eps = sampler_table(sched, method, eta=eta, logsnr_lag=lag)
        v, f_v = sampler_table(sched, method, eta=eta, logsnr_lag=lag, prediction='v')
        a = S.alphas_cumprod()[np.asarray(sched.timesteps)[::-1]]
        np.testing.assert_allclose(v[:, C_RECIP], np.sqrt(a), rtol=1e-15, atol=0)
        np.testing.assert_allclose(v[:, C_RECIPM1], np.sqrt(1. - a), rtol=1e-15, atol=0)
        assert np.array_equal(v[:, 2:], eps[:, 2:]) and f_v == f_eps
        assert np.array_equal(eps, sampler_table(sched, method, eta=eta, logsnr_lag=lag, prediction='eps')[0])
    assert (v[:, C_RECIP] ** 2 + v[:, C_RECIPM1] ** 2 == pytest.approx(1.0, abs=1e-15))


def _x0_fp32(row, z, out):
    """The step kernels' unclipped x0 = c_recip z - c_recipm1 out, with the fp32 table entries and fp32 arithmetic."""
    r = row.astype(np.float32)
    return (r[C_RECIP] * z - r[C_RECIPM1] * out).astype(np.float32)


@pytest.mark.parametrize('t', [0, 1, 10, 300, 700, 990, 998, 999])
def test_oracle_denoiser_recovers_x0_and_v_does_not_amplify_errors(t):
    sched = Schedule(1000)
    k = 999 - t                                                         # loop position of timestep t
    eps_row, v_row = sampler_table(sched)[0][k], sampler_table(sched, prediction='v')[0][k]
    ac = S.alphas_cumprod()[t]
    alpha, sigma = np.sqrt(ac), np.sqrt(1. - ac)
    rng = np.random.RandomState(t)
    x0 = rng.uniform(-1, 1, 4096)
    eps = rng.randn(4096)
    z = alpha * x0 + sigma * eps
    v = alpha * eps - sigma * x0
    # exact predictions through the fp32 formula recover x0 to fp32 rounding of the terms it sums
    z32 = z.astype(np.float32)
    for row, out in ((v_row, v), (eps_row, eps)):
        got = _x0_fp32(row, z32, out.astype(np.float32)).astype(np.float64)
        scale = abs(np.float32(row[C_RECIP])) * np.abs(z) + abs(np.float32(row[C_RECIPM1])) * np.abs(out) + np.abs(x0)
        assert (np.abs(got - x0) <= 4 * np.finfo(np.float32).eps * scale).all(), (t, row[:2])
    # a perturbation delta of the prediction: the unclipped x0 moves by -sigma delta (v) and -sqrt(1/abar - 1) delta (eps)
    delta = 1e-3 * rng.randn(4096)
    for row, out, gain in ((v_row, v, sigma), (eps_row, eps, np.sqrt(1. / ac - 1.))):
        err = (row[C_RECIP] * z - row[C_RECIPM1] * (out + delta)) - (row[C_RECIP] * z - row[C_RECIPM1] * out)
        np.testing.assert_allclose(err, -gain * delta, rtol=1e-9, atol=1e-15 * row[C_RECIP] * np.abs(z).max())
    assert sigma <= 1.0
    if t == 999:
        assert np.sqrt(1. / ac - 1.) > 6e4                             # the eps path's gain at the first sampling step


def test_v_target_restates_the_formula_in_fp32():
    B, S_ = 6, 8
    rng = np.random.RandomState(3)
    x0 = rng.uniform(-1, 1, (B, S_, S_, 3)).astype(np.float32)
    noise = rng.randn(B, S_, S_, 3).astype(np.float32)
    t = np.array([0, 1, 500, 990, 998, 999])
    sa, sb = diffusion_tables()
    assert sa.dtype == sb.dtype == np.float32 and sa.shape == sb.shape == (1000,)
    ac = S.alphas_cumprod()
    np.testing.assert_allclose(sa, np.sqrt(ac), rtol=2 ** -24, atol=0)
    np.testing.assert_allclose(sb, np.sqrt(1. - ac), rtol=2 ** -24, atol=0)
    got = v_target(x0, noise, t)
    assert got.dtype == np.float32
    for b in range(B):
        a, s = np.float32(sa[t[b]]), np.float32(sb[t[b]])
        want = np.float32(a * noise[b]) - np.float32(s * x0[b])     # each product and the difference rounded once in fp32
        assert np.array_equal(got[b].view(np.int32), want.astype(np.float32).view(np.int32)), b
    # z = alpha x0 + sigma eps and v give back x0 = alpha z - sigma v and eps = sigma z + alpha v (fp64)
    a64, s64 = np.sqrt(ac[t])[:, None, None, None], np.sqrt(1. - ac[t])[:, None, None, None]
    z = a64 * x0 + s64 * noise
    v = a64 * noise - s64 * x0
    np.testing.assert_allclose(a64 * z - s64 * v, x0, atol=1e-12)
    np.testing.assert_allclose(s64 * z + a64 * v, noise, atol=1e-12)


@pytest.mark.parametrize('gamma', [1.0, 5.0, 20.0])
def test_min_snr_weights_of_v(gamma):
    ac = S.alphas_cumprod()
    snr = ac / (1. - ac)
    v = min_snr_weights(gamma, prediction='v')
    np.testing.assert_allclose(v, np.minimum(snr, gamma) / (snr + 1.), rtol=1e-14, atol=0)
    assert np.array_equal(min_snr_weights(gamma), min_snr_weights(gamma, prediction='eps'))
    np.testing.assert_allclose(min_snr_weights(gamma), np.minimum(snr, gamma) / snr, rtol=1e-14, atol=0)
    assert (v <= 1.0).all() and (v > 0).all()


def test_unknown_or_unsupported_predictions_are_rejected():
    assert PREDICTIONS == ('eps', 'v')
    for bad in ('x0', 'V', None):
        with pytest.raises(ValueError):
            sampler_table(Schedule(10), prediction=bad)
        with pytest.raises(ValueError):
            min_snr_weights(5.0, prediction=bad)
        with pytest.raises(ValueError):
            create_train_state(0, 1, 1e-4, 2, 16, prediction=bad, loss='mse')
    for loss in ('frobenius',):
        with pytest.raises(ValueError, match="loss='mse'"):
            create_train_state(0, 1, 1e-4, 2, 16, prediction='v', loss=loss)
    with pytest.raises(ValueError, match="loss='mse'"):
        create_train_state(0, 1, 1e-4, 2, 16, prediction='v')                  # the default loss is the Frobenius norm
    for m in METHODS:
        assert sampler_table(Schedule(10), m, prediction='v')[0].shape == (10, 8)


def test_prediction_round_trips_through_the_checkpoint(tmp_path):
    src = _state(1, 3, step=4)
    src.prediction = 'v'
    path = ck.save_train_state(str(tmp_path), src, step=4)
    raw = ck.msgpack_restore(open(path, 'rb').read())
    assert raw['prediction'] == 'v'
    assert ck.parse_train_state_tree(raw, SPEC, N)['prediction'] == 'v'
    dst = _state(2, 4)
    dst.prediction = 'v'
    assert ck.restore_train_state(str(tmp_path), dst) is dst
    assert torch.equal(dst.params.flat, src.params.flat) and dst.step == 4
    # a file of the other prediction is refused before anything is written
    eps = _state(5, 4)
    before = eps.params.flat.clone()
    with pytest.raises(ValueError, match='prediction'):
        ck.restore_train_state(str(tmp_path), eps)
    assert torch.equal(eps.params.flat, before) and eps.step == 0
    # the file is still a plain params checkpoint for the sampler
    params = ck.restore_checkpoint(str(tmp_path), prefix='state')
    assert set(params) == {'Conv_0', 'GroupNorm_0'}
    # an eps state writes 'eps'
    ck.save_train_state(str(tmp_path / 'e'), _state(1, 3, step=2), step=2)
    assert ck.msgpack_restore(open(tmp_path / 'e' / 'state2', 'rb').read())['prediction'] == 'eps'


def test_checkpoints_without_a_prediction_read_as_eps(tmp_path):
    """Files written before v-prediction existed: they restore into an eps state and are refused by a v one."""
    p, m, v, e = (np.random.RandomState(s).randn(N).astype(np.float32) for s in range(4))
    tree = ck.train_state_tree(ck.leaf_tree(p, SPEC), ck.leaf_tree(m, SPEC), ck.leaf_tree(v, SPEC), count=3, step=3)
    assert 'prediction' not in tree
    ck.save_checkpoint(str(tmp_path), tree, step=3, prefix='state')
    assert ck.parse_train_state_tree(tree, SPEC, N)['prediction'] == 'eps'
    dst = _state(7, 1, ema=False)
    assert dst.prediction == 'eps'
    with pytest.warns(UserWarning):                                       # the file holds no cond_mask streams
        ck.restore_train_state(str(tmp_path), dst)
    assert np.array_equal(dst.params.flat.numpy(), p) and dst.step == 3
    vst = _state(7, 1, ema=False)
    vst.prediction = 'v'
    with pytest.raises(ValueError, match='prediction'):
        ck.restore_train_state(str(tmp_path), vst)
