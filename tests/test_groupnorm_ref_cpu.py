"""CPU checks of tests/groupnorm_ref.py, the fp64 reference the GroupNorm kernels are held to: the forward against
torch.nn.functional.group_norm and the oracle, every backward stage formula against torch autograd."""
import pytest
import torch
import torch.nn.functional as F

from oracle import xunet_ref as R
from tests import groupnorm_ref as G
from tests.util import keep_mask


def _inputs(N, H, W, C, seed, film=False, shift=0.):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, C, generator=g, dtype=torch.float64) * 1.7 + shift
    gamma = 1. + 0.3 * torch.randn(C, generator=g, dtype=torch.float64)
    beta = 0.2 * torch.randn(C, generator=g, dtype=torch.float64)
    e = 0.5 * torch.randn(N, H, W, 2 * C, generator=g, dtype=torch.float64) if film else None
    return x, gamma, beta, e


@pytest.mark.parametrize('shape', [(2, 4, 4, 32), (4, 8, 6, 96), (6, 2, 3, 64)])
def test_forward_plain_matches_torch_group_norm_on_the_joint_frame_view(shape):
    N, H, W, C = shape
    x, gamma, beta, _ = _inputs(N, H, W, C, 1)
    got = G.forward(x, gamma, beta, G.PLAIN)
    # (N, H, W, C) -> (B, C, 2H, W): both frames of a sample stacked along one spatial axis
    xv = x.reshape(N // 2, 2, H, W, C).permute(0, 4, 1, 2, 3).reshape(N // 2, C, 2 * H, W)
    ref = F.group_norm(xv, 32, gamma, beta, eps=G.EPS)
    ref = ref.reshape(N // 2, C, 2, H, W).permute(0, 2, 3, 4, 1).reshape(N, H, W, C)
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)


def test_statistics_from_sums_match_two_pass_statistics():
    x, gamma, beta, _ = _inputs(4, 6, 5, 96, 2)
    m0, r0 = G.mean_rstd(x)
    m1, r1 = G.mean_rstd_from_sums(G.group_sums(G.cstats(x)), 6, 5, 96)
    assert torch.allclose(m0, m1, rtol=1e-12, atol=1e-12) and torch.allclose(r0, r1, rtol=1e-10)
    t = G.table(m0, r0, gamma, beta)
    xh = G.xhat(x, m0, r0)
    # the table's affine form is the normalisation
    assert torch.allclose(x * t[..., 0].repeat_interleave(2, 0)[:, None, None] + t[..., 1].repeat_interleave(2, 0)[:, None, None],
                          xh, atol=1e-12)


@pytest.mark.parametrize('mode', [G.PLAIN, G.SWISH])
def test_forward_matches_oracle_group_norm(mode):
    N, H, W, C = 4, 4, 4, 64
    x, gamma, beta, _ = _inputs(N, H, W, C, 3)
    ref = R.group_norm(x.reshape(N // 2, 2, H, W, C), {'GroupNorm_0': {'scale': gamma, 'bias': beta}}).reshape(N, H, W, C)
    if mode == G.SWISH:
        ref = R.swish(ref)
    assert torch.allclose(G.forward(x, gamma, beta, mode), ref, rtol=1e-12, atol=1e-12)


def test_film_matches_oracle_film():
    N, H, W, C, E = 2, 4, 4, 32, 8
    x, gamma, beta, _ = _inputs(N, H, W, C, 4)
    g = torch.Generator().manual_seed(5)
    emb = torch.randn(N, H, W, E, generator=g, dtype=torch.float64)
    p = {'Dense_0': {'kernel': torch.randn(E, 2 * C, generator=g, dtype=torch.float64) * 0.3,
                     'bias': torch.randn(2 * C, generator=g, dtype=torch.float64) * 0.1}}
    e = R.dense(R.swish(emb), p['Dense_0'])           # the stored FiLM tensor [scale | shift]
    yhat = G.forward(x, gamma, beta, G.PLAIN)
    ref = R.swish(R.film(yhat, emb, p))
    assert torch.allclose(G.forward(x, gamma, beta, G.FILM, e=e), ref, rtol=1e-12, atol=1e-12)


def test_resampling_matches_oracle():
    x, gamma, beta, _ = _inputs(2, 6, 4, 32, 6)
    a = G.forward(x, gamma, beta, G.SWISH)
    down = R.avgpool_downsample(a.reshape(1, 2, 6, 4, 32)).reshape(2, 3, 2, 32)
    up = R.nearest_neighbor_upsample(a.reshape(1, 2, 6, 4, 32)).reshape(2, 12, 8, 32)
    assert torch.allclose(G.forward(x, gamma, beta, G.SWISH, G.RS_DOWN), down, atol=1e-14)
    assert torch.allclose(G.forward(x, gamma, beta, G.SWISH, G.RS_UP), up, atol=1e-14)


def test_dropout_mask_index_is_the_element_index():
    m = torch.from_numpy(keep_mask(7, 3, (2, 4, 4, 32), 0.25))
    assert m.shape == (2, 4, 4, 32) and 0.6 < m.double().mean() < 0.9
    x, gamma, beta, e = _inputs(2, 4, 4, 32, 7, film=True)
    full = G.forward(x, gamma, beta, G.FILM, e=e)
    dropped = G.forward(x, gamma, beta, G.FILM, e=e, keep=m, drop_rate=0.25)
    assert torch.all(dropped[~m] == 0)
    assert torch.allclose(dropped[m], full[m] / 0.75, rtol=1e-7)


BWD_CASES = [(G.PLAIN, G.RS_NONE, False), (G.SWISH, G.RS_NONE, False), (G.FILM, G.RS_NONE, False), (G.FILM, G.RS_NONE, True),
             (G.PLAIN, G.RS_DOWN, False), (G.SWISH, G.RS_DOWN, False), (G.PLAIN, G.RS_UP, False), (G.SWISH, G.RS_UP, False)]


@pytest.mark.parametrize('mode,rs,drop', BWD_CASES)
def test_backward_stage_formulas_match_autograd(mode, rs, drop):
    N, H, W, C = 4, 4, 6, 64
    x, gamma, beta, e = _inputs(N, H, W, C, 10 + mode * 3 + rs, film=mode == G.FILM, shift=0.4)
    keep = torch.from_numpy(keep_mask(99, 2, (N, H, W, C), 0.3)) if drop else None
    leaves = [t.clone().requires_grad_(True) for t in (x, gamma, beta)] + ([e.clone().requires_grad_(True)] if e is not None else [])
    out = G.forward(leaves[0], leaves[1], leaves[2], mode, rs, e=leaves[3] if e is not None else None, keep=keep, drop_rate=0.3)
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    (out * gout).sum().backward()

    mean, rstd = G.mean_rstd(x)
    xh = G.xhat(x, mean, rstd)
    dyh, de = G.dyhat(G.resample_adjoint(gout, rs), x, gamma, beta, mode, e=e, keep=keep, drop_rate=0.3)
    sums = G.bcs(dyh, xh)
    dx, scale = G.dx(dyh, xh, rstd, gamma, sums)
    dgamma, dbeta = G.dgamma_dbeta(sums)
    assert torch.allclose(dx, leaves[0].grad, rtol=1e-9, atol=1e-11 * float(scale.max()))
    assert torch.allclose(dgamma, leaves[1].grad, rtol=1e-10, atol=1e-10)
    assert torch.allclose(dbeta, leaves[2].grad, rtol=1e-10, atol=1e-10)
    if mode == G.FILM:
        assert torch.allclose(de, leaves[3].grad, rtol=1e-10, atol=1e-12)
