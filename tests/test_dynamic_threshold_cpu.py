"""Dynamic thresholding without a GPU: the order-statistic restatement of the per-view scale equals np.quantile bit for bit,
the thresholded fp64 steps reduce to tests/solver_ref.py's when s = 1, and the Sampler's argument check."""
import math

import numpy as np
import pytest
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.sampling import _check_dynamic_threshold
from tests import solver_ref as S
from tests import threshold_ref as T

PERCENTILES = (0.5, 0.9, 0.995, 1.0)


def _views(per, rng):
    """fp32 |x0|-like views of `per` values: continuous, heavily tied, all equal, with zeros, and of wide dynamic range."""
    yield np.abs(rng.standard_normal(per) * 3).astype(np.float32)
    yield np.abs(np.round(rng.standard_normal(per) * 2)).astype(np.float32)
    yield np.full(per, 2.5, np.float32)
    v = np.abs(rng.standard_normal(per)).astype(np.float32)
    v[rng.random(per) < 0.6] = 0.0
    yield v
    yield np.abs(rng.standard_normal(per) * 10.0 ** rng.uniform(-6, 6, per)).astype(np.float32)


@pytest.mark.parametrize('per', [1, 2, 7, 12288, 49152])
def test_order_statistic_is_numpy_quantile(per):
    rng = np.random.default_rng(per)
    for k, a in enumerate(_views(per, rng)):
        for p in PERCENTILES:
            ref = np.quantile(a.astype(np.float64), p)
            got = T.quantile_linear(a, p)
            assert np.float64(got).tobytes() == np.float64(ref).tobytes(), (k, p, got, ref)
            s = T.threshold_scale(a, p)
            assert s == max(np.float32(ref), np.float32(1.0)) and s.dtype == np.float32


def test_threshold_is_the_clip_when_s_is_one():
    x0 = torch.tensor([[-3.0, -0.5, 0.25, 0.75], [0.5, -0.9, 0.1, 0.0]], dtype=torch.float64)
    out, s = T.threshold(x0, 0.5)
    assert s.tolist() == [max(1.0, float(np.quantile([3.0, 0.5, 0.25, 0.75], 0.5))), 1.0]
    assert torch.equal(out[1], x0[1])
    big, sb = T.threshold(x0 * 10, 0.75)
    assert (sb > 1).all() and float(big.abs().max()) <= 1.0


def _small_inputs(g, n=4096, B=4):
    """eps and z small enough that every view's x0 stays inside [-1, 1] at moderate noise (s = 1)."""
    return [(torch.randn(B, n // B, generator=g, dtype=torch.float64) * 0.1) for _ in range(4)]


@pytest.mark.parametrize('method', ['ddpm', 'ddim', 'dpmpp_2m'])
def test_threshold_steps_reduce_to_solver_ref(method):
    ac = S.alphas_cumprod()
    ts = [300, 200, 100, 0]
    g = torch.Generator().manual_seed(2)
    x0_prev = x0r_prev = None
    for k, t in enumerate(ts):
        ec, eu, z, nz = _small_inputs(g)
        ac_next = ac[ts[k + 1]] if k + 1 < len(ts) else 1.0
        if method == 'ddpm':
            got, x0, s = T.ddpm_step(ec, eu, z, ac[t], ac_next, nz, 0.995)
            ref, x0r = S.ddim_step(ec, eu, z, ac[t], ac_next, nz, eta=1.0)      # DDIM at eta = 1 is the DDPM posterior
            assert torch.allclose(got, ref, rtol=1e-12, atol=1e-14), k
        elif method == 'ddim':
            got, x0, s = T.ddim_step(ec, eu, z, ac[t], ac_next, nz, 0.995, eta=0.5)
            ref, x0r = S.ddim_step(ec, eu, z, ac[t], ac_next, nz, eta=0.5)
            assert torch.equal(got, ref), k
        else:
            prev_ac = ac[ts[k - 1]] if k else None
            got, x0, s = T.dpmpp_2m_step(ec, eu, z, ac[t], ac_next, x0_prev, prev_ac, 0.995)
            ref, x0r = S.dpmpp_2m_step(ec, eu, z, ac[t], ac_next, x0r_prev, prev_ac)
            assert torch.equal(got, ref), k
            x0_prev, x0r_prev = x0, x0r
        assert (s == 1.0).all() and torch.equal(x0, x0r), k


def test_thresholding_changes_the_step_when_s_exceeds_one():
    ac = S.alphas_cumprod()
    g = torch.Generator().manual_seed(3)
    ec, eu, z = (torch.randn(2, 768, generator=g, dtype=torch.float64) for _ in range(3))
    got, x0, s = T.ddim_step(ec, eu, z, ac[900], ac[800], 0.0, 0.995)
    ref, x0r = S.ddim_step(ec, eu, z, ac[900], ac[800], 0.0)
    assert (s > 1).all() and float(x0.abs().max()) <= 1.0 and not torch.allclose(got, ref)


@pytest.mark.parametrize('p', [0, 0.0, -0.5, 1.0000001, 2, float('nan'), float('inf'), '0.9', True])
def test_bad_dynamic_threshold_is_rejected(p):
    with pytest.raises(ValueError):
        _check_dynamic_threshold(p)
    # the Sampler checks it before it touches the model or the device
    with pytest.raises(ValueError):
        P.Sampler(None, None, 1, 16, steps=6, dynamic_threshold=p)


@pytest.mark.parametrize('p', [None, 1e-6, 0.5, 0.995, 1.0, 1, np.float32(0.9)])
def test_good_dynamic_threshold_is_accepted(p):
    _check_dynamic_threshold(p)
    assert p is None or 0.0 < float(p) <= 1.0 and not math.isnan(float(p))
