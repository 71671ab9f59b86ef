"""Consistency distillation without a GPU: `consistency_grid`, the consistency sampler table, `cd_target_table`, the
fixed point of the training target on the exact denoiser of Gaussian data (teacher step -> target network -> target
formula returns the teacher's DDIM chain f(z, n) for every n), multistep consistency sampling with f, argument validation,
and the consistency-distillation record in the training-state checkpoint."""
import math

import numpy as np
import pytest
import torch

from novel_view_synthesis_3d_b200 import checkpoint as ck
from novel_view_synthesis_3d_b200 import distill as D
from novel_view_synthesis_3d_b200.sampling import (METHODS, SAMPLER_METHODS, Sampler, Schedule, consistency_grid,
                                                   distill_grid, logsnr_schedule_cosine, sampler_table)
from tests import cd_ref as R
from tests import solver_ref as SR
from tests.test_distill_cpu import _student, _teacher
from tests.test_train_state_checkpoint import N as NPARAMS, SPEC, _state


# ---- the sampling grid ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [2, 16, 50, 256, 1000])
def test_consistency_grid_nests_in_the_teacher_grid(n):
    g = distill_grid(n, 0)
    assert len(g) == n
    for k in sorted({min(k, n) for k in (1, 2, 3, 4, 7, n // 2, n)}):
        c = consistency_grid(n, k)
        assert len(c) == k and c[0] == g[0] == 999 and np.all(np.diff(c) < 0)
        assert np.array_equal(c, g[(np.arange(k) * n) // k]) and set(c) <= set(g)
    assert np.array_equal(consistency_grid(n, n), g)


def test_consistency_grid_arguments():
    for n, k in [(16, 0), (16, 17), (0, 1), (-3, 1), (16, 1.5), (16, True), (2.5, 1)]:
        with pytest.raises(ValueError):
            consistency_grid(n, k)


# ---- the sampler table ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('pred', ['eps', 'v'])
@pytest.mark.parametrize('n,k', [(16, 1), (16, 4), (256, 2), (256, 4), (64, 64)])
def test_consistency_rows(pred, n, k):
    ts = consistency_grid(n, k)
    rows, first = sampler_table(Schedule(timesteps=ts), 'consistency', prediction=pred)
    ac = SR.alphas_cumprod()
    a = ac[ts]
    a1 = np.append(ac[ts[1:]], 1.0)
    assert rows.shape == (k, 8)
    np.testing.assert_allclose(rows[:, R.C_X0], np.sqrt(a1), rtol=1e-14, atol=0)
    np.testing.assert_allclose(rows[:, R.SIGMA], np.sqrt(1. - a1), rtol=1e-14, atol=0)
    assert (rows[:, R.C_Z] == 0).all() and (rows[:, R.C_PREV] == 0).all() and (rows[:, 7] == 0).all()
    # the last row lands on x0: z' = x0
    assert rows[-1, R.C_X0] == 1.0 and rows[-1, R.SIGMA] == 0.0
    want = (np.sqrt(1. / a), np.sqrt(1. / a - 1.)) if pred == 'eps' else (np.sqrt(a), np.sqrt(1. - a))
    np.testing.assert_allclose(rows[:, R.C_RECIP], want[0], rtol=1e-14)
    np.testing.assert_allclose(rows[:, R.C_RECIPM1], want[1], rtol=1e-14)
    # the lag is off by default: each forward sees the log-SNR of the timestep z is at
    assert first == logsnr_schedule_cosine(ts[0] / 1000)
    np.testing.assert_array_equal(rows[:-1, R.LOGSNR], logsnr_schedule_cosine(ts[1:] / 1000))
    assert sampler_table(Schedule(timesteps=ts), 'consistency', prediction=pred, logsnr_lag=True)[1] == -20.0


def test_the_teacher_methods_keep_their_tables():
    """METHODS stays the teacher samplers, and their tables keep the reference lag by default."""
    assert METHODS == ('ddpm', 'ddim', 'dpmpp_2m') and SAMPLER_METHODS == METHODS + ('consistency',)
    for m in METHODS:
        for s in (Schedule(50), Schedule(25, spacing='logsnr')):
            a, b = sampler_table(s, m), sampler_table(s, m, logsnr_lag=True)
            assert np.array_equal(a[0], b[0]) and a[1] == b[1] == -20.0
    with pytest.raises(ValueError, match='eta'):
        sampler_table(Schedule(16), 'consistency', eta=0.5)
    with pytest.raises(ValueError, match='eta'):
        Sampler(None, None, 1, 16, method='consistency', eta=1.0)
    with pytest.raises(ValueError, match='unknown sampler method'):
        sampler_table(Schedule(16), 'lcm')


# ---- the target table -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [2, 16, 256])
def test_cd_target_table_matches_fp64(n):
    g = distill_grid(n, 0)
    tab = D.cd_target_table(g)
    ac = SR.alphas_cumprod()
    assert tab.shape == (n, 4) and tab.dtype == np.float64
    for i in range(n):
        a1 = ac[g[i + 1]] if i + 1 < n else 1.0
        want = (math.sqrt(a1), math.sqrt(1. - a1), math.sqrt(ac[g[i]]), math.sqrt(1. - ac[g[i]]))
        np.testing.assert_allclose(tab[i], want, rtol=1e-14, atol=0)
    assert tab[-1, 0] == 1.0 and tab[-1, 1] == 0.0


# ---- the fixed point on the exact denoiser --------------------------------------------------------------------------------------
@pytest.mark.parametrize('teacher_pred', ['eps', 'v'])
@pytest.mark.parametrize('w', [0.5, None])
@pytest.mark.parametrize('n', [16, 50])
def test_the_target_of_a_perfect_student_is_its_own_output(teacher_pred, w, n):
    """With the target network equal to f(., n+1), the teacher's DDIM chain to clean, the fp64 teacher step -> target
    network at the row's log-SNR -> target formula gives a v* with alpha_n z - sigma_n v* = f(z, n), for every n including
    the last (the boundary, where x0- is the teacher's clipped x0).  An off-by-one in the rows, the log-SNR column or the
    boundary breaks it."""
    grid = distill_grid(n, 0)
    ttab, first = sampler_table(Schedule(timesteps=grid), 'ddim', prediction=teacher_pred, logsnr_lag=False)
    gtab = D.cd_target_table(grid)
    teacher = R.teacher_fn(teacher_pred, w)
    ac = SR.alphas_cumprod()
    assert first == logsnr_schedule_cosine(grid[0] / 1000)
    r = np.random.RandomState(n)
    for i in range(n):
        a = ac[grid[i]]
        z = math.sqrt(a) * (0.1 + 0.2 * r.randn(128)) + math.sqrt(1. - a) * r.randn(128)
        seen = []

        def target_net(z_hat, logsnr):
            k = R.position_of_logsnr(grid, logsnr)
            seen.append(k)
            return R.student_v(z_hat, k, grid, ttab, teacher)
        v, z_hat, _ = R.cd_target(z, i, grid, ttab, gtab, teacher, target_net)
        assert seen == [min(i + 1, n - 1)]
        f = R.ddim_chain(z, i, grid, ttab, teacher)
        np.testing.assert_allclose(math.sqrt(a) * z - math.sqrt(1. - a) * v, f, rtol=0, atol=1e-12)
        if i == n - 1:
            np.testing.assert_array_equal(z_hat, f)           # the last teacher row lands on its clipped x0


@pytest.mark.parametrize('n', [16, 64])
def test_one_consistency_step_of_f_is_the_teachers_ddim_sample(n):
    """K = 1: the consistency sampler with the perfect student f gives the teacher's N-step DDIM sample (solver_ref's
    independent fp64 DDIM on the exact denoiser); K = 4 gives the chain re-noised at each sampling timestep."""
    grid = distill_grid(n, 0)
    ttab, _ = sampler_table(Schedule(timesteps=grid), 'ddim', prediction='eps', logsnr_lag=False)
    teacher = R.teacher_fn('eps', None)
    r = np.random.RandomState(7)
    z_T = r.randn(256)
    pos = {t: i for i, t in enumerate(grid)}
    for k in (1, 4):
        ts = consistency_grid(n, k)
        rows, _ = sampler_table(Schedule(timesteps=ts), 'consistency', prediction='v')
        noises = r.randn(k, 256)
        got = R.consistency_sample(z_T, ts, rows, lambda z, j: R.student_v(z, pos[ts[j]], grid, ttab, teacher), noises)
        if k == 1:
            want = SR.run_exact('ddim', grid[::-1], torch.as_tensor(z_T)).numpy()
        else:
            ac, z = SR.alphas_cumprod(), z_T
            for j in range(k):
                x0 = R.ddim_chain(z, pos[ts[j]], grid, ttab, teacher)
                a1 = ac[ts[j + 1]] if j + 1 < k else 1.0
                z = math.sqrt(a1) * x0 + math.sqrt(1. - a1) * noises[j]
            want = z
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-11)


# ---- argument validation --------------------------------------------------------------------------------------------------------
def _cd_teacher(**kw):
    """A ConsistencyTeacher's attributes without its engine (check_teacher reads only these)."""
    t = object.__new__(D.ConsistencyTeacher)
    for key, v in vars(_teacher(**kw)).items():
        setattr(t, key, v)
    return t


def test_arguments_are_validated():
    data = object()
    D.check_teacher(_student(), _cd_teacher(grid=distill_grid(7, 0)), data)      # any N >= 2, odd included
    for skw, match in [(dict(prediction='eps'), "prediction='v'"), (dict(loss='frobenius'), "loss='mse'"),
                       (dict(reference_quirks=True), 'reference_quirks'), (dict(batch_size=4), 'B = ')]:
        with pytest.raises(ValueError, match=match):
            D.check_teacher(_student(**skw), _cd_teacher(), data)
    with pytest.raises(ValueError, match='data='):
        D.check_teacher(_student(), _cd_teacher(), None)
    # a progressive-distillation teacher keeps its even-grid check
    with pytest.raises(ValueError, match='odd'):
        D.check_teacher(_student(), _teacher(grid=distill_grid(7, 0)), data)
    for kw, match in [(dict(steps=1), 'N >= 2'), (dict(w=-1.0), 'w must'), (dict(w=float('inf')), 'w must'),
                      (dict(prediction='x0'), 'prediction')]:
        args = dict(steps=16, batch_size=2, img_sidelength=16)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            D.ConsistencyTeacher(None, None, args.pop('steps'), **args)


def test_cd_record_round_trips_through_the_checkpoint(tmp_path):
    for rec in ({'cd_steps': 64, 'w': 3.0}, {'cd_steps': 50}):
        d = tmp_path / str(len(rec))
        src = _state(1, 3, step=4)
        src.prediction, src.distill = 'v', rec
        path = ck.save_train_state(str(d), src, step=4)
        got = ck.parse_train_state_tree(ck.msgpack_restore(open(path, 'rb').read()), SPEC, NPARAMS)['distill']
        assert got == rec and type(got['cd_steps']) is int
        dst = _state(2, 4)
        dst.prediction, dst.distill = 'v', dict(rec)
        assert ck.restore_train_state(str(d), dst) is dst
        assert torch.equal(dst.params.flat, src.params.flat) and dst.step == 4
        for other in ({'cd_steps': 32, 'w': 3.0}, {'cd_steps': 64, 'w': 2.0}, {'teacher_steps': 64, 'rounds': 1}, None):
            if other == rec:
                continue
            st = _state(5, 4)
            st.prediction, st.distill = 'v', other
            with pytest.raises(ValueError, match='distillation record'):
                ck.restore_train_state(str(d), st)
            assert st.step == 0


def test_the_examples_read_n_from_the_state_checkpoint(tmp_path):
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'examples'))
    from distill_srn import cd_steps
    with pytest.raises(FileNotFoundError):
        cd_steps(str(tmp_path))
    st = _state(1, 3, step=2)
    st.prediction, st.distill = 'v', {'cd_steps': 48, 'w': 3.0}
    ck.save_train_state(str(tmp_path), st, step=2)
    st.distill = {'cd_steps': 64, 'w': 3.0}
    path = ck.save_train_state(str(tmp_path), st, step=7)
    assert cd_steps(str(tmp_path)) == 64 and cd_steps(path) == 64
    st.distill = {'teacher_steps': 256, 'rounds': 1}
    ck.save_train_state(str(tmp_path / 'pd'), st, step=1)
    with pytest.raises(ValueError, match='consistency'):
        cd_steps(str(tmp_path / 'pd'))
