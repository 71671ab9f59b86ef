"""The mean-squared epsilon loss without a GPU: the reference loss against its closed form, the min-SNR-gamma weight table,
and the argument checks of the training API."""
import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.diffusion import min_snr_weights
from novel_view_synthesis_3d_b200.train import check_accum_batch, check_loss_weight
from novel_view_synthesis_3d_b200.xunet import check_loss
from tests.mse_ref import mse_loss

B, S = 3, 4
P_ELEMS = S * S * 3


def _residuals(seed=0):
    g = torch.Generator().manual_seed(seed)
    eps = torch.randn(B, S, S, 3, generator=g, dtype=torch.float64)
    noise = torch.randn(B, S, S, 3, generator=g, dtype=torch.float64)
    return eps, noise


@pytest.mark.parametrize('w', [None, [0.5, 2.0, 1.25]])
def test_mse_loss_is_the_weighted_mean_of_squares_and_its_gradient_is_closed_form(w):
    eps, noise = _residuals()
    eps.requires_grad_(True)
    loss = mse_loss(eps, noise, None if w is None else torch.tensor(w, dtype=torch.float64))
    wb = np.ones(B) if w is None else np.asarray(w)
    r = (eps.detach() - noise).numpy().reshape(B, -1)
    assert float(loss.detach()) == pytest.approx(float(np.mean(wb * (r ** 2).mean(axis=1))), rel=1e-14)
    (g,) = torch.autograd.grad(loss, eps)
    want = 2.0 * wb[:, None] * r / (B * P_ELEMS)
    np.testing.assert_allclose(g.numpy().reshape(B, -1), want, rtol=1e-13, atol=0)


def test_zero_weight_removes_a_sample():
    eps, noise = _residuals(1)
    eps.requires_grad_(True)
    loss = mse_loss(eps, noise, torch.tensor([1.0, 0.0, 1.0], dtype=torch.float64))
    (g,) = torch.autograd.grad(loss, eps)
    assert bool((g[1] == 0).all()) and bool((g[0] != 0).any())
    moved = noise.clone()
    moved[1] += 100.0                                     # sample 1 no longer counts, whatever its error
    assert float(mse_loss(eps.detach(), moved, torch.tensor([1.0, 0.0, 1.0], dtype=torch.float64))) == float(loss.detach())


@pytest.mark.parametrize('gamma', [1.0, 5.0])
def test_min_snr_weights_follow_the_cosine_beta_table(gamma):
    ac = np.cumprod(1.0 - P.cosine_beta_schedule(1000), axis=0)
    snr = ac / (1.0 - ac)
    w = min_snr_weights(gamma)
    assert w.shape == (1000,) and w.dtype == np.float64
    np.testing.assert_array_equal(w, np.minimum(snr, gamma) / snr)
    assert (w > 0).all() and (w <= 1).all()
    assert w[0] < 1e-3 and w[-1] == 1.0                   # t = 0 is nearly noise-free; t = 999 is nearly pure noise
    assert np.all(np.diff(w) >= 0)                         # the SNR falls with t, so the weight rises to 1


@pytest.mark.parametrize('gamma', [0.0, -1.0, float('nan'), float('inf')])
def test_min_snr_gamma_must_be_positive_and_finite(gamma):
    with pytest.raises(ValueError):
        min_snr_weights(gamma)


@pytest.mark.parametrize('loss', ['l1', 'MSE', '', None])
def test_unknown_loss_is_rejected(loss):
    with pytest.raises(ValueError):
        check_loss(loss)
    with pytest.raises(ValueError):
        P.create_train_state(0, 1, 1e-4, 2, 16, loss=loss)      # rejected before any device work


def test_known_losses_pass():
    assert check_loss('frobenius') == 'frobenius' and check_loss('mse') == 'mse'


def test_weights_need_the_mse_loss():
    with pytest.raises(ValueError, match="loss='mse'"):
        check_loss_weight('frobenius', np.ones(2, np.float32), 2)
    check_loss_weight('frobenius', None, 2)
    check_loss_weight('mse', None, 2)
    check_loss_weight('mse', np.array([0.0, 3.5], np.float32), 2)
    check_loss_weight('mse', torch.tensor([0.0, 3.5]), 2)


@pytest.mark.parametrize('w', [[1.0, -0.5], [1.0, float('nan')], [float('inf'), 1.0], [-0.0, -1e-30]])
def test_negative_or_non_finite_host_weights_are_rejected(w):
    with pytest.raises(ValueError, match='finite'):
        check_loss_weight('mse', np.asarray(w, np.float32), 2)
    with pytest.raises(ValueError, match='finite'):
        check_loss_weight('mse', torch.tensor(w), 2)


@pytest.mark.parametrize('shape', [(3,), (1,), (2, 1), ()])
def test_weights_of_the_wrong_shape_are_rejected(shape):
    with pytest.raises(ValueError, match='shape'):
        check_loss_weight('mse', np.ones(shape, np.float32), 2)


def test_accumulation_checks_the_rows_of_the_weights():
    k, b = 2, 3
    batch = {key: np.zeros((k * b,) + shp, np.float32) for key, shp in
             [('x', (S, S, 3)), ('z', (S, S, 3)), ('logsnr', ()), ('R1', (3, 3)), ('t1', (3,)), ('R2', (3, 3)),
              ('t2', (3,)), ('K', (3, 3))]}
    noise = np.zeros((k * b, S, S, 3), np.float32)
    check_accum_batch(batch, noise, None, k, b, np.ones(k * b, np.float32))
    with pytest.raises(ValueError, match='loss_weight'):
        check_accum_batch(batch, noise, None, k, b, np.ones(b, np.float32))
    check_loss_weight('mse', np.ones(k * b, np.float32), k * b)
    with pytest.raises(ValueError):
        check_loss_weight('mse', np.ones(b, np.float32), k * b)
