"""Progressive distillation without a GPU: the nested grids of `distill_grid`, `Schedule(timesteps=..)`, the target
algebra on the exact denoiser of Gaussian data (one student DDIM step fed the v target lands on the teacher's two-step
z''), argument validation, and the distillation record in the training-state checkpoint."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from novel_view_synthesis_3d_b200 import checkpoint as ck
from novel_view_synthesis_3d_b200 import distill as D
from novel_view_synthesis_3d_b200.sampling import METHODS, Schedule, distill_grid, sampler_table
from novel_view_synthesis_3d_b200.train import TrainStep
from novel_view_synthesis_3d_b200.xunet import XUNetConfig
from tests import solver_ref as S
from tests.test_train_state_checkpoint import N, SPEC, _state

C_RECIP, C_RECIPM1, C_X0, C_Z, SIGMA, LOGSNR = range(6)


@pytest.mark.parametrize('steps', [256, 64, 512])
def test_distill_grid_nests(steps):
    g0 = distill_grid(steps, 0)
    assert np.array_equal(g0, Schedule(steps).timesteps[::-1])
    prev = g0
    for r in range(1, 5):
        g = distill_grid(steps, r)
        assert np.array_equal(g, prev[0::2]) and g[0] == 999 and len(g) == len(g0) >> r
        assert np.all(np.diff(g) < 0)
        prev = g
    assert len(distill_grid(256, 8)) == 1
    with pytest.raises(ValueError, match='odd'):
        distill_grid(256, 9)
    with pytest.raises(ValueError, match='odd'):
        distill_grid(250, 2)                      # 250 -> 125 -> ?
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError, match='rounds'):
            distill_grid(256, bad)


@pytest.mark.parametrize('steps', [256, 1000, 25])
def test_schedule_of_explicit_timesteps_is_bit_identical(steps):
    ref, ex = Schedule(steps), Schedule(timesteps=Schedule(steps).timesteps)
    rev = Schedule(timesteps=Schedule(steps).timesteps[::-1])           # any order
    for m, eta in [(m, 0.0) for m in METHODS] + [('ddim', 1.0)]:
        for pred in ('eps', 'v'):
            for lag in (True, False):
                a = sampler_table(ref, m, eta=eta, prediction=pred, logsnr_lag=lag)
                for s in (ex, rev):
                    b = sampler_table(s, m, eta=eta, prediction=pred, logsnr_lag=lag)
                    assert np.array_equal(a[0], b[0]) and a[1] == b[1]
    for bad in ([], [3, 3], [-1, 5], [10, 1000], [[1, 2]], [0.5, 2.0]):
        with pytest.raises(ValueError, match='timesteps'):
            Schedule(timesteps=bad)


def _exact_out(z, ac, prediction, mu, s):
    """The exact eps (or v) of per-pixel Gaussian data N(mu, s^2) at alpha-bar ac."""
    eps = S.exact_eps(z, ac, mu=mu, s=s)
    if prediction == 'eps':
        return eps
    x0 = (z - math.sqrt(1. - ac) * eps) / math.sqrt(ac)
    return math.sqrt(ac) * eps - math.sqrt(1. - ac) * x0


def _step(row, out, z):
    """The fixed-clip table step in fp64 (sigma = 0 rows); returns (z_next, x0 before the clip)."""
    x0 = row[C_RECIP] * z - row[C_RECIPM1] * out
    return row[C_X0] * np.clip(x0, -1., 1.) + row[C_Z] * z, x0


@pytest.mark.parametrize('teacher_pred', ['eps', 'v'])
@pytest.mark.parametrize('w', [0.5, None])
@pytest.mark.parametrize('steps,rounds', [(64, 0), (256, 2)])
def test_student_step_on_the_target_lands_on_the_teachers_two_steps(teacher_pred, w, steps, rounds):
    """For every student row m, including the last interval (to x0): the teacher's two DDIM steps from z_t, with the exact
    conditional denoiser (guided against a different "unconditional" one when w is set), give z''; the v target of
    target_table fed to the student's DDIM v table row m gives z'' again, to 1e-12."""
    grid = distill_grid(steps, rounds)
    ac_full = S.alphas_cumprod()
    ttab, _ = sampler_table(Schedule(timesteps=grid), 'ddim', prediction=teacher_pred, logsnr_lag=False)
    stab, _ = sampler_table(Schedule(timesteps=grid[0::2]), 'ddim', prediction='v', logsnr_lag=False)
    gtab = D.target_table(grid)
    assert ttab.shape == (len(grid), 8) and stab.shape == gtab[:, :1].shape[:1] + (8,) and len(gtab) == len(grid) // 2
    r = np.random.RandomState(steps + rounds)
    for m in range(len(grid) // 2):
        t, t1 = grid[2 * m], grid[2 * m + 1]
        ac = ac_full[t]
        x0 = 0.1 + 0.2 * r.randn(256)
        z = math.sqrt(ac) * x0 + math.sqrt(1. - ac) * r.randn(256)

        def teacher(zz, tt):
            a = ac_full[tt]
            oc = _exact_out(zz, a, teacher_pred, S.MU, S.SD)
            if w is None:
                return oc
            return (1 + w) * oc - w * _exact_out(zz, a, teacher_pred, -0.05, 0.25)
        z1, xa = _step(ttab[2 * m], teacher(z, t), z)
        z2, xb = _step(ttab[2 * m + 1], teacher(z1, t1), z1)
        assert np.abs(xa).max() < 1 and np.abs(xb).max() < 1            # the clip is inactive
        c_a, c_b, alpha, sigma = gtab[m]
        assert alpha == math.sqrt(ac) and sigma == math.sqrt(1. - ac)
        xt = c_a * z2 - c_b * z
        v = (alpha * z - xt) / sigma
        zs, xs = _step(stab[m], v, z)
        assert np.abs(xs).max() < 1
        np.testing.assert_allclose(zs, z2, rtol=0, atol=1e-12)
        if m == len(grid) // 2 - 1:
            assert c_a == 1.0 and c_b == 0.0 and np.array_equal(xt, z2)  # the last interval: x~ = z'' = x0'


def test_teacher_rows_are_one_sampler_step_each():
    """Row 2m of the teacher table steps G_T[2m] -> G_T[2m+1] and hands the next forward log-SNR(G_T[2m+1])."""
    grid = distill_grid(32, 0)
    tab, first = sampler_table(Schedule(timesteps=grid), 'ddim', prediction='eps', logsnr_lag=False)
    ac = S.alphas_cumprod()
    from novel_view_synthesis_3d_b200.sampling import logsnr_schedule_cosine
    assert first == logsnr_schedule_cosine(grid[0] / 1000)
    for k in range(len(grid) - 1):
        assert tab[k, LOGSNR] == logsnr_schedule_cosine(grid[k + 1] / 1000)
        a, a1 = ac[grid[k]], ac[grid[k + 1]]
        assert math.isclose(tab[k, C_Z], math.sqrt((1 - a1) / (1 - a)), rel_tol=1e-14)
    assert tab[-1, C_X0] == 1.0 and tab[-1, C_Z] == 0.0


def _teacher(**kw):
    t = dict(S=16, B=2, grid=distill_grid(8, 0), model=SimpleNamespace(config=XUNetConfig()), device='cuda:0')
    t.update(kw)
    return SimpleNamespace(**t)


def _student(**kw):
    s = dict(prediction='v', loss='mse', reference_quirks=False, img_sidelength=16, batch_size=2,
             model=SimpleNamespace(config=XUNetConfig()), params=SimpleNamespace(flat=SimpleNamespace(device='cuda:0')))
    s.update(kw)
    return SimpleNamespace(**s)


def test_arguments_are_validated():
    data = object()
    D.check_teacher(_student(), _teacher(), data)
    cases = [(dict(), dict(), None, 'data='),
             (dict(prediction='eps'), dict(), data, "prediction='v'"),
             (dict(loss='frobenius'), dict(), data, "loss='mse'"),
             (dict(reference_quirks=True), dict(), data, 'reference_quirks'),
             (dict(), dict(grid=np.arange(7)), data, 'odd'),
             (dict(img_sidelength=32), dict(), data, 'S = '),
             (dict(batch_size=4), dict(), data, 'B = '),
             (dict(model=SimpleNamespace(config=XUNetConfig(ch=64))), dict(), data, 'model'),
             (dict(params=SimpleNamespace(flat=SimpleNamespace(device='cuda:1'))), dict(), data, 'lives on')]
    for skw, tkw, d, match in cases:
        with pytest.raises(ValueError, match=match):
            D.check_teacher(_student(**skw), _teacher(**tkw), d)
    # TrainStep checks before it builds anything
    with pytest.raises(ValueError, match='data='):
        TrainStep(_student(), teacher=_teacher())
    with pytest.raises(ValueError, match='min_snr_gamma'):
        TrainStep(_student(), data=data, teacher=_teacher(), min_snr_gamma=5.0)
    # Teacher arguments (checked before the engine is built)
    for kw, match in [(dict(w=-1.0), 'w must'), (dict(w=float('nan')), 'w must'), (dict(prediction='x0'), 'prediction'),
                      (dict(rounds=1), 'distilled student'), (dict(rounds=1, w=None), 'distilled student'),
                      (dict(steps=250, rounds=1, w=None, prediction='v'), 'odd')]:
        args = dict(steps=64, batch_size=2, img_sidelength=16)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            D.Teacher(None, None, args.pop('steps'), **args)
    with pytest.raises(ValueError, match='even'):
        D.target_table(np.arange(5))


def test_distill_record_round_trips_through_the_checkpoint(tmp_path):
    rec = {'teacher_steps': 256, 'rounds': 1, 'w': 3.0}
    src = _state(1, 3, step=4)
    src.prediction, src.distill = 'v', rec
    path = ck.save_train_state(str(tmp_path), src, step=4)
    raw = ck.msgpack_restore(open(path, 'rb').read())
    assert ck.parse_train_state_tree(raw, SPEC, N)['distill'] == rec
    dst = _state(2, 4)
    dst.prediction, dst.distill = 'v', dict(rec)
    assert ck.restore_train_state(str(tmp_path), dst) is dst
    assert torch.equal(dst.params.flat, src.params.flat) and dst.step == 4
    # another round, guidance or teacher grid -- or a plain v model -- is refused before anything is written
    for other in ({'teacher_steps': 256, 'rounds': 2}, {'teacher_steps': 128, 'rounds': 1, 'w': 3.0},
                  {'teacher_steps': 256, 'rounds': 1, 'w': 2.0}, None):
        st = _state(5, 4)
        st.prediction, st.distill = 'v', other
        before = st.params.flat.clone()
        with pytest.raises(ValueError, match='distillation record'):
            ck.restore_train_state(str(tmp_path), st)
        assert torch.equal(st.params.flat, before) and st.step == 0
    # an unguided round (no 'w') round-trips too
    src.distill = {'teacher_steps': 256, 'rounds': 2}
    ck.save_train_state(str(tmp_path / 'u'), src, step=5)
    assert ck.parse_train_state_tree(ck.msgpack_restore(open(tmp_path / 'u' / 'state5', 'rb').read()), SPEC, N)['distill'] \
        == {'teacher_steps': 256, 'rounds': 2}


def test_files_without_a_record_are_not_distilled(tmp_path):
    """Files written before distillation existed, and files of plain models, carry no record: they restore into a state
    without one and are refused by a student."""
    ck.save_train_state(str(tmp_path), _state(1, 3, step=2), step=2)
    raw = ck.msgpack_restore(open(tmp_path / 'state2', 'rb').read())
    assert 'distill' not in raw and ck.parse_train_state_tree(raw, SPEC, N)['distill'] is None
    assert ck.restore_train_state(str(tmp_path), _state(2, 3)).distill is None
    st = _state(2, 3)
    st.distill = {'teacher_steps': 256, 'rounds': 1, 'w': 3.0}
    with pytest.raises(ValueError, match='distillation record'):
        ck.restore_train_state(str(tmp_path), st)
