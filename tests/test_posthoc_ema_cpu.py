"""Post-hoc EMA without a GPU: sigma_rel <-> gamma, the weights of the power-average recursion, the fp64 solve against the
restatement in tests/posthoc_ref.py, reconstruction of other EMA lengths in a synthetic run, argument errors, and the
snapshot and train-state records."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from novel_view_synthesis_3d_b200 import checkpoint as ck
from novel_view_synthesis_3d_b200 import posthoc as ph
from tests import posthoc_ref as R

SPEC = {'Conv_0/kernel': ((1, 3, 3, 3, 4), 0), 'Conv_0/bias': ((4,), 108),
        'GroupNorm_0/GroupNorm_0/scale': ((4,), 112), 'GroupNorm_0/GroupNorm_0/bias': ((4,), 116)}
N = 120


# ---- sigma_rel <-> gamma ---------------------------------------------------------------------------------------------------
def test_pinned_gammas():
    assert ph.sigma_rel_to_gamma(0.05) == pytest.approx(16.9722, abs=5e-5)
    assert ph.sigma_rel_to_gamma(0.10) == pytest.approx(6.9372, abs=5e-5)


@pytest.mark.parametrize('sr', [0.01, 0.03, 0.05, 0.075, 0.1, 0.15, 0.2, 0.28])
def test_sigma_rel_gamma_round_trip(sr):
    g = ph.sigma_rel_to_gamma(sr)
    assert g > 0
    assert ph.gamma_to_sigma_rel(g) == pytest.approx(sr, rel=1e-12)
    assert g == pytest.approx(R.gamma_of(sr), rel=1e-9)


# ---- the recursion ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('gamma', [0.5, 6.9372, 16.9722])
@pytest.mark.parametrize('T', [1, 2, 37, 1000])
def test_recursion_weights_are_the_closed_form(gamma, T):
    w = R.recursion_weights(T, gamma)
    assert w[0] == 0.0                                       # beta_1 = 0: no weight on the initial parameters
    np.testing.assert_allclose(w, R.closed_form_weights(T, gamma), rtol=1e-10, atol=1e-15)
    assert w.sum() == pytest.approx(1.0, abs=1e-12)


def test_solve_matches_the_restatement():
    in_t = [100, 100, 300, 300, 1000, 1000]
    in_g = [6.9372, 16.9722] * 3
    c = ph.solve_coefficients(in_t, in_g, 700, 10.0)
    np.testing.assert_allclose(c, R.coefficients(in_t, in_g, 700, 10.0), rtol=1e-6, atol=1e-9)
    # arrays of targets give one column each
    cc = ph.solve_coefficients(in_t, in_g, [700, 1000], [10.0, 3.0])
    assert cc.shape == (6, 2)
    np.testing.assert_allclose(cc[:, 0], c, rtol=1e-12)


# ---- reconstruction in a synthetic run (T = 20000 updates, snapshots of both averages every 1000) ---------------------------
@pytest.fixture(scope='module')
def synthetic():
    T, every = 20000, 1000
    theta = R.trajectory(T)
    gammas = [ph.sigma_rel_to_gamma(0.05), ph.sigma_rel_to_gamma(0.10)]
    return theta, gammas, R.run_averages(theta, gammas, every)


def _reconstruct(snaps, t, g):
    c = ph.solve_coefficients([s[0] for s in snaps], [s[1] for s in snaps], t, g)
    return sum(ci * s[2] for ci, s in zip(c, snaps)), c


@pytest.mark.parametrize('k', [0, 1])
def test_a_tracked_profile_returns_its_snapshot(synthetic, k):
    theta, gammas, snaps = synthetic
    T = snaps[-1][0]
    got, c = _reconstruct(snaps, T, gammas[k])
    one_hot = np.zeros(len(snaps))
    one_hot[len(snaps) - 2 + k] = 1.0
    np.testing.assert_allclose(c, one_hot, atol=1e-9)
    want = snaps[len(snaps) - 2 + k][2]
    assert np.linalg.norm(got - want) <= 1e-12 * np.linalg.norm(want)


@pytest.mark.parametrize('sr', [0.03, 0.075, 0.15])
def test_other_lengths_are_reconstructed(synthetic, sr):
    theta, gammas, snaps = synthetic
    T = snaps[-1][0]
    g = ph.sigma_rel_to_gamma(sr)
    got, _ = _reconstruct(snaps, T, g)
    want = R.exact_average(theta, T, g)
    nearer = min(np.linalg.norm(want - R.exact_average(theta, T, gk)) for gk in gammas)
    err = np.linalg.norm(got - want)
    assert err <= 1e-2 * nearer, (sr, err / nearer)


# ---- argument errors ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bad', [0.0, -0.1, ph.SIGMA_REL_MAX, 0.3, float('nan'), float('inf')])
def test_sigma_rel_out_of_range(bad):
    with pytest.raises(ValueError):
        ph.sigma_rel_to_gamma(bad)


@pytest.mark.parametrize('bad', [-1.0, -2.0, float('nan'), float('inf')])
def test_gamma_out_of_range(bad):
    with pytest.raises(ValueError):
        ph.gamma_to_sigma_rel(bad)


@pytest.mark.parametrize('bad', [(0.05,), (0.05, 0.1, 0.15), (0.05, 0.05), (0.05, 0.3), 0.05, (0.0, 0.1)])
def test_posthoc_option_errors(bad):
    with pytest.raises(ValueError):
        ph.check_posthoc_ema(bad)


def test_solve_argument_errors():
    with pytest.raises(ValueError):
        ph.solve_coefficients([], [], 10, 5.0)
    with pytest.raises(ValueError):
        ph.solve_coefficients([10, 20], [5.0], 10, 5.0)
    with pytest.raises(ValueError):
        ph.solve_coefficients([0, 20], [5.0, 6.0], 10, 5.0)
    with pytest.raises(ValueError):
        ph.solve_coefficients([10, 20], [5.0, -1.0], 10, 5.0)
    with pytest.raises(ValueError):
        ph.solve_coefficients([10, 20], [5.0, 6.0], 10, float('nan'))


def test_create_train_state_rejects_ema_decay_with_posthoc():
    from novel_view_synthesis_3d_b200 import create_train_state
    with pytest.raises(ValueError, match='exclusive'):
        create_train_state(0, 1, 1e-4, 1, 64, ema_decay=0.999, posthoc_ema=(0.05, 0.1))
    with pytest.raises(ValueError):
        create_train_state(0, 1, 1e-4, 1, 64, posthoc_ema=(0.05, 0.5))


# ---- snapshots ---------------------------------------------------------------------------------------------------------------
def _fake_state(count, seed, sigma_rel=(0.05, 0.1), spec=SPEC, n=N):
    r = np.random.RandomState(seed)
    a, b = (torch.from_numpy(r.randn(n).astype(np.float32)) for _ in range(2))
    post = SimpleNamespace(a=SimpleNamespace(flat=a), b=SimpleNamespace(flat=b), sigma_rel=sigma_rel,
                           gamma=tuple(ph.sigma_rel_to_gamma(s) for s in sigma_rel), flats=lambda: [a, b])
    return SimpleNamespace(posthoc=post, params=SimpleNamespace(spec=spec), opt_state=SimpleNamespace(count=count))


def test_snapshot_round_trip_and_reconstruct(tmp_path):
    states = [_fake_state(c, c) for c in (300, 100, 200)]
    for s in states:
        ph.save_snapshot(str(tmp_path), s)
    snaps = ph.load_snapshots(str(tmp_path))
    assert [s.t for s in snaps] == [100, 200, 300]
    by_t = {s.opt_state.count: s for s in states}
    for s in snaps:
        st = by_t[s.t]
        assert s.sigma_rel == (0.05, 0.1) and s.gamma == st.posthoc.gamma
        a, b = s.averages()
        np.testing.assert_array_equal(a['Conv_0']['kernel'].reshape(-1), st.posthoc.a.flat[:108].numpy())
        np.testing.assert_array_equal(b['GroupNorm_0']['GroupNorm_0']['bias'], st.posthoc.b.flat[116:].numpy())
        assert a['Conv_0']['kernel'].dtype == np.float32
    # reconstruct on the CPU: the fp64 sum of the coefficients times the snapshots, rounded once
    sr = 0.075
    g = ph.sigma_rel_to_gamma(sr)
    c = R.coefficients([t for t in (100, 200, 300) for _ in range(2)], [x for _ in range(3) for x in states[0].posthoc.gamma],
                       250, g)
    want = sum(c[2 * i] * by_t[t].posthoc.a.flat.double().numpy() + c[2 * i + 1] * by_t[t].posthoc.b.flat.double().numpy()
               for i, t in enumerate((100, 200, 300)))
    tree = ph.reconstruct(str(tmp_path), sr, t=250, device='cpu')
    got = ck.leaf_tree(np.zeros(N, np.float32), SPEC)
    flat = np.concatenate([np.asarray(tree['Conv_0']['kernel']).reshape(-1), tree['Conv_0']['bias'],
                           tree['GroupNorm_0']['GroupNorm_0']['scale'], tree['GroupNorm_0']['GroupNorm_0']['bias']])
    assert flat.dtype == np.float32 and got.keys() == tree.keys()
    np.testing.assert_allclose(flat, want, rtol=2 ** -23, atol=1e-6 * np.abs(want).max())
    # the default t is the last snapshot's, where the first tracked width is its snapshot
    last = ph.reconstruct(str(tmp_path), 0.05, device='cpu')
    np.testing.assert_allclose(last['Conv_0']['bias'], by_t[300].posthoc.a.flat[108:112].numpy(), rtol=1e-6, atol=1e-6)


def test_snapshot_errors(tmp_path):
    with pytest.raises(FileNotFoundError):
        ph.load_snapshots(str(tmp_path))
    with pytest.raises(ValueError):
        ph.save_snapshot(str(tmp_path), SimpleNamespace(posthoc=None))
    ph.save_snapshot(str(tmp_path), _fake_state(100, 1))
    with pytest.raises(ValueError, match='outside'):
        ph.reconstruct(str(tmp_path), 0.08, t=101, device='cpu')
    spec2 = dict(SPEC)
    spec2['Conv_0/bias'] = ((5,), 108)
    ph.save_snapshot(str(tmp_path), _fake_state(200, 2, spec=spec2, n=N + 1))
    with pytest.raises(ValueError, match='not of one model'):
        ph.load_snapshots(str(tmp_path))


# ---- the train-state record ------------------------------------------------------------------------------------------------
def test_train_state_record_round_trip():
    r = np.random.RandomState(0)
    p, m, v, a, b = (r.randn(N).astype(np.float32) for _ in range(5))
    lt = lambda x: ck.leaf_tree(x, SPEC)
    for axis in (False, True):
        tree = ck.train_state_tree(lt(p), lt(m), lt(v), count=9, step=9, add_device_axis=axis,
                                   posthoc=(lt(a), lt(b)), posthoc_sigma_rel=(0.05, 0.1))
        raw = ck.msgpack_restore(ck.msgpack_serialize(tree))
        assert raw['posthoc_sigma_rel'].dtype == np.float64 and raw['posthoc_sigma_rel'].shape == (2,)
        out = ck.parse_train_state_tree(raw, SPEC, N)
        assert out['posthoc_sigma_rel'] == (0.05, 0.1)
        np.testing.assert_array_equal(out['posthoc'][0].numpy(), a)
        np.testing.assert_array_equal(out['posthoc'][1].numpy(), b)
        np.testing.assert_array_equal(out['params'].numpy(), p)
    # a file without the averages parses as before
    out = ck.parse_train_state_tree(ck.msgpack_restore(ck.msgpack_serialize(
        ck.train_state_tree(lt(p), lt(m), lt(v), count=3, step=3))), SPEC, N)
    assert out['posthoc'] is None and out['posthoc_sigma_rel'] is None
