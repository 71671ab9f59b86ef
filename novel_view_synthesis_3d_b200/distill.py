"""Progressive distillation (Salimans & Ho 2022, Alg. 2) on this project's discrete cosine schedule.

A student is trained to take one DDIM step for two of its teacher's.  The teacher samples with DDIM (eta = 0) on a grid G_T of
2N timesteps in loop order (`sampling.distill_grid`); the student's grid is G_S = G_T[0::2], and its step m runs from
t = G_T[2m] to t'' = G_T[2m+2] ("clean" after the last) through the teacher's midpoint t' = G_T[2m+1].  For one sample:

    m ~ U{0..N-1}, t = G_S[m], z_t = alpha_t x0 + sigma_t eps          (xunet_srn_batch_distill)
    z_t'  = DDIM step of the teacher from z_t, row 2m of its table       (teacher forward, xunet_distill_teacher_step)
    z_t'' = DDIM step of the teacher from z_t', row 2m+1                 (teacher forward, xunet_distill_target)
    x~ = (z_t'' - (sigma''/sigma_t) z_t) / (alpha'' - (sigma''/sigma_t) alpha_t),   v = (alpha_t z_t - x~) / sigma_t,

and the student, a v-prediction model trained with loss='mse' (the paper's "SNR + 1" weighting), regresses its conditional
output at (z_t, log-SNR(t)) onto v.  A student DDIM step whose output is v lands exactly on z_t''.  A guided teacher (w a
float, the original 3DiM model) runs the 2B batch [cond ; uncond] and steps (1 + w) out_c - w out_u; the student learns the
guided result as a conditional model, so it is sampled with Sampler(w=None), one B-batch forward per step.  The student of
one round is the unguided teacher (w=None) of the next.

    teacher = Teacher(model, params, 256, batch_size=B, img_sidelength=S, w=3.0)
    state = create_distill_state(teacher, learning_rate=1e-4)
    step = TrainStep(state, data=store, teacher=teacher)     # every draw, teacher forward and target inside the step graph

Consistency distillation (Song et al. 2023, Consistency Models, Alg. 2; `ConsistencyTeacher`) trains a 1-4-step student in one
run against the original guided teacher: its target is the student's own x0 prediction one teacher DDIM step further down
the teacher grid (see ConsistencyTeacher), and it is sampled with Sampler(method='consistency', w=None, prediction='v',
timesteps=consistency_grid(N, K)).  The same create_distill_state and TrainStep(data=, teacher=) train it.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from . import dist as xdist
from .sampling import Schedule, check_prediction, cosine_beta_schedule, distill_grid, sampler_table
from .xunet import XUNet, Engine, ParamTree, pack_flat


def target_table(grid) -> np.ndarray:
    """The per-student-row target coefficients (N, 4) float64 of a teacher grid G_T of 2N timesteps in loop order: row m =
    {c_a, c_b, alpha_t, sigma_t} with t = G_T[2m], t'' = G_T[2m+2] (alpha'' = 1, sigma'' = 0 after the last),
    c_a = 1 / (alpha'' - (sigma''/sigma_t) alpha_t) and c_b = (sigma''/sigma_t) c_a, so x~ = c_a z'' - c_b z_t and
    v = (alpha_t z_t - x~) / sigma_t."""
    g = np.asarray(grid, dtype=np.int64)
    if len(g) % 2:
        raise ValueError(f'a teacher grid has an even number of timesteps, got {len(g)}')
    ac = np.cumprod(1. - cosine_beta_schedule(1000), axis=0)
    a = ac[g[0::2]]
    a2 = np.concatenate([ac[g[2::2]], [1.0]])
    alpha, sigma, alpha2, sigma2 = np.sqrt(a), np.sqrt(1. - a), np.sqrt(a2), np.sqrt(1. - a2)
    r = sigma2 / sigma
    c_a = 1. / (alpha2 - r * alpha)
    return np.stack([c_a, r * c_a, alpha, sigma], 1)


def cd_target_table(grid) -> np.ndarray:
    """The consistency-distillation target coefficients (N, 4) float64 of a teacher grid G of N timesteps in loop order:
    row n = {a, b, alpha_n, sigma_n} with alpha_n, sigma_n those of t_n = G[n], a = alpha_{n+1} and b = sigma_{n+1} of
    t_{n+1} = G[n+1], and (a, b) = (1, 0) on the last row (t_{n+1} = clean), so that x0- = clip(a z^ - b v-) and
    v* = (alpha_n z_t - x0-) / sigma_n."""
    g = np.asarray(grid, dtype=np.int64)
    ac = np.cumprod(1. - cosine_beta_schedule(1000), axis=0)
    a, a1 = ac[g], np.concatenate([ac[g[1:]], [1.0]])
    return np.stack([np.sqrt(a1), np.sqrt(1. - a1), np.sqrt(a), np.sqrt(1. - a)], 1)


def _check_teacher_args(prediction, w) -> Optional[float]:
    """The prediction and guidance weight of a teacher; returns w as a float (or None)."""
    check_prediction(prediction)
    if w is not None:
        w = float(w)
        if not (np.isfinite(w) and w >= 0.0):
            raise ValueError(f'w must be a finite number >= 0 (or None for an unguided teacher), got {w}')
    return w


class _FrozenTeacher:
    """What both teachers hold: the model, its own inference engine of copies * B rows ([cond ; uncond] when guided, cond_mask
    set once), a copy of the parameters, the DDIM table of `grid`, the target table, the grid positions the draw picks t
    from and the per-sample positions m, all in device memory.  The subclasses validate their arguments first."""

    def __init__(self, model: XUNet, params, steps: int, grid, batch_size: int, img_sidelength: int, w: Optional[float],
                 prediction: str, target_rows, grid_t):
        self.prediction = prediction
        self.model, self.steps, self.w, self.grid = model, int(steps), w, grid
        self.B, self.S = int(batch_size), int(img_sidelength)
        self.copies = 1 if w is None else 2
        self.eng = Engine(model.config, self.copies * self.B, self.S, False, model.device)
        self.device = self.eng.device
        if isinstance(params, ParamTree) and getattr(params, 'flat', None) is not None:
            if params.flat.numel() != self.eng.nparams:
                raise ValueError(f'the teacher parameters hold {params.flat.numel()} values, the model at S = {self.S} has '
                                 f'{self.eng.nparams}')
            self.flat = params.flat.detach().to(self.device, torch.float32).clone()
        else:
            self.flat = pack_flat(params, self.eng.spec, self.eng.nparams).to(self.device)
        rows, _ = sampler_table(Schedule(timesteps=grid), 'ddim', prediction=prediction, logsnr_lag=False)
        self.table_rows, self.target_rows = rows, target_rows
        f32 = dict(dtype=torch.float32, device=self.device)
        self.table = torch.as_tensor(rows, **f32)
        self.target = torch.as_tensor(self.target_rows, **f32)
        self.grid_t = torch.as_tensor(grid_t, dtype=torch.int32, device=self.device)
        self.m = torch.zeros(self.B, dtype=torch.int32, device=self.device)
        self.eng.inp['cond_mask'].copy_(torch.cat([torch.ones(self.B), torch.zeros((self.copies - 1) * self.B)]))


class Teacher(_FrozenTeacher):
    """A frozen teacher for progressive distillation, and the device state one distillation step reads.

    model, params: the teacher network (a Flax-layout tree or a ParamTree; the parameters are copied, so the teacher stays
    fixed whatever happens to `params` later).  steps, rounds: the teacher samples with DDIM on
    `distill_grid(steps, rounds)`, i.e. it is the original model (rounds = 0) or a student distilled `rounds` times from a
    `steps`-step teacher; its student then samples on `distill_grid(steps, rounds + 1)` (`student_grid`).
    w: the guidance weight of a guided teacher (2B batch [cond ; uncond]); None for a teacher without guidance, such as a
    student of an earlier round, which must then be given w=None.  prediction: what the teacher predicts, 'eps' or 'v'.
    batch_size, img_sidelength: the student's micro-batch and image side.

    It owns its own inference engine (not shared with a Sampler of the same model), the teacher's DDIM table
    (`sampler_table(Schedule(timesteps=grid), 'ddim', prediction=prediction, logsnr_lag=False)`, 2N rows), the target
    table (`target_table`), the student grid and the per-sample grid positions m, all in device memory."""

    def __init__(self, model: XUNet, params, steps: int, *, batch_size: int, img_sidelength: int,
                 w: Optional[float] = 3.0, prediction: str = 'eps', rounds: int = 0):
        w = _check_teacher_args(prediction, w)
        grid = distill_grid(steps, rounds)
        if len(grid) % 2:
            raise ValueError(f'the teacher grid distill_grid({steps}, {rounds}) has odd length {len(grid)}: its '
                             f'student cannot take one step for two')
        if rounds > 0 and (w is not None or prediction != 'v'):
            raise ValueError(f'a teacher of round {rounds} is a distilled student: a v-prediction model without guidance '
                             f"(w=None, prediction='v'), got w={w}, prediction={prediction!r}")
        self.rounds = int(rounds)
        self.student_grid = grid[0::2].copy()
        super().__init__(model, params, steps, grid, batch_size, img_sidelength, w, prediction, target_table(grid),
                         self.student_grid)

    @property
    def record(self) -> dict:
        """What a student's checkpoint records of its distillation: the original teacher's step count, the student's round
        and the guidance weight this teacher applied (absent when it applied none)."""
        r = {'teacher_steps': self.steps, 'rounds': self.rounds + 1}
        if self.w is not None:
            r['w'] = self.w
        return r


class ConsistencyTeacher(_FrozenTeacher):
    """A frozen teacher for consistency distillation (Song et al. 2023, Consistency Models, Alg. 2, with a guided teacher as
    in LCM), and the device state one consistency-distillation step reads.

    model, params, w, prediction, batch_size, img_sidelength: as for `Teacher` (an original model: no rounds).  steps: the
    teacher grid is G = distill_grid(steps, 0) of N timesteps in loop order (any N >= 2); the student is trained at every
    position n of it and sampled on `sampling.consistency_grid(N, K)` with method='consistency'.  One training sample is

        n ~ U{0..N-1}, z = alpha_n x0 + sigma_n eps                    (xunet_srn_batch_distill on G)
        z^ = DDIM step of the teacher from z, row n of its table         (teacher forward, xunet_cd_teacher_step)
        v- = the student's own output at (z^, log-SNR(t_{n+1}))          (the target network: the current weights, mu = 0,
                                                                          no dropout, on the student's training engine)
        x0- = clip(alpha_{n+1} z^ - sigma_{n+1} v-) (x0- = z^ for n = N-1),   v* = (alpha_n z - x0-) / sigma_n
                                                                         (xunet_cd_target, `cd_target_table`)

    and the student regresses its v output at (z, log-SNR(t_n)) onto v*: the consistency loss
    ||f(z, t_n) - f-(z^, t_{n+1})||^2 of f(z, t) = alpha_t z - sigma_t v, weighted SNR + 1 in x0.

    It owns, besides what `Teacher` owns (an N-row DDIM table here), the device scratch of the target forward: z^ (B, S, S, 3),
    its log-SNRs (B) and v- (B, S, S, 3)."""

    def __init__(self, model: XUNet, params, steps: int, *, batch_size: int, img_sidelength: int,
                 w: Optional[float] = 3.0, prediction: str = 'eps'):
        w = _check_teacher_args(prediction, w)
        grid = distill_grid(steps, 0)
        if len(grid) < 2:
            raise ValueError(f'consistency distillation needs a teacher grid of N >= 2 timesteps, distill_grid({steps}, 0) '
                             f'has {len(grid)}')
        super().__init__(model, params, steps, grid, batch_size, img_sidelength, w, prediction, cd_target_table(grid), grid)
        f32 = dict(dtype=torch.float32, device=self.device)
        self.z_hat = torch.zeros(self.B, self.S, self.S, 3, **f32)
        self.logsnr_hat = torch.zeros(self.B, **f32)
        self.v_minus = torch.zeros(self.B, self.S, self.S, 3, **f32)

    @property
    def record(self) -> dict:
        """What a student's checkpoint records of its consistency distillation: the teacher grid's N and the guidance weight
        this teacher applied (absent when it applied none)."""
        r = {'cd_steps': len(self.grid)}
        if self.w is not None:
            r['w'] = self.w
        return r


def create_distill_state(teacher: _FrozenTeacher, learning_rate: float = 1e-4, *, rng_dropout=None, ema_decay: Optional[float] = None,
                         max_grad_norm: Optional[float] = None, warmup_steps: int = 0, posthoc_ema: Optional[tuple] = None):
    """The TrainState of a student of `teacher` (a Teacher or a ConsistencyTeacher): the teacher's model, batch size and image side, prediction='v' with
    loss='mse', and parameters (and EMA or post-hoc averages, when kept) starting from the teacher's.  The state records teacher.record, which
    save_train_state writes and restore_train_state checks.  The optimizer arguments are create_train_state's."""
    from .train import create_train_state
    st = create_train_state(0, rng_dropout, learning_rate, teacher.B, teacher.S, model=teacher.model, init_on_device=True,
                            ema_decay=ema_decay, max_grad_norm=max_grad_norm, warmup_steps=warmup_steps, loss='mse',
                            prediction='v', posthoc_ema=posthoc_ema)
    st.params.flat.copy_(teacher.flat)
    if st.ema_params is not None:
        st.ema_params.flat.copy_(teacher.flat)
    if st.posthoc is not None:
        for f in st.posthoc.flats():
            f.copy_(teacher.flat)
    st.distill = teacher.record
    return st


def _draw(step, j: int) -> None:
    """The distillation draw of micro-batch j: slot j and the teacher's rows, t on the teacher's grid_t, m in T.m."""
    T, d, lib = step.teacher, step.data, step.lib
    st = torch.cuda.current_stream(step.dev).cuda_stream
    _lib.check(lib.xunet_srn_batch_distill(C.byref(d.c_store), step.step_dev.data_ptr(), step.data_seed, j, step.k,
                                           xdist.rank(), step.world, T.B, step.sqrt_ac.data_ptr(), step.sqrt_1mac.data_ptr(),
                                           T.grid_t.data_ptr(), len(T.grid_t), C.byref(step.inputs.cbatch[j]),
                                           C.byref(T.eng.cbatch), T.copies, T.m.data_ptr(), None, None, st),
               'xunet_srn_batch_distill')


def run_teacher(step, j: int) -> None:
    """Micro-batch j of a distillation TrainStep, all on the current stream: the draw, the teacher forwards and steps, and
    the v target in slot j's noise segment (progressive distillation: the teacher's two steps; consistency distillation:
    the teacher's step and the target forward of the student's own weights on its training engine)."""
    T, inp, lib = step.teacher, step.inputs.inp[j], step.lib
    st = torch.cuda.current_stream(step.dev).cuda_stream
    B, per = T.B, T.S * T.S * 3
    w = 0.0 if T.w is None else T.w
    _draw(step, j)
    T.eng.forward(T.flat, train=False)
    if isinstance(T, ConsistencyTeacher):
        _lib.check(lib.xunet_cd_teacher_step(T.eng.eps.data_ptr(), w, T.copies, T.table.data_ptr(), T.m.data_ptr(), B, per,
                                             inp['z'].data_ptr(), T.z_hat.data_ptr(), T.logsnr_hat.data_ptr(), st),
                   'xunet_cd_teacher_step')
        # the target network: slot j's conditioning at (z^, log-SNR(t_{n+1})), without dropout.  The student's train forward
        # follows on the same engine and rewrites everything the backward reads
        cb = _lib.XunetBatch.from_buffer_copy(step.inputs.cbatch[j])
        cb.z, cb.logsnr = T.z_hat.data_ptr(), T.logsnr_hat.data_ptr()
        step.eng.forward(step.state.params.flat, train=False, batch=cb, out=T.v_minus)
        _lib.check(lib.xunet_cd_target(T.v_minus.data_ptr(), T.target.data_ptr(), T.m.data_ptr(), inp['z'].data_ptr(),
                                       T.z_hat.data_ptr(), B, per, inp['noise'].data_ptr(), st), 'xunet_cd_target')
        return
    _lib.check(lib.xunet_distill_teacher_step(T.eng.eps.data_ptr(), w, T.copies, T.table.data_ptr(), T.m.data_ptr(), B, per,
                                              C.byref(T.eng.cbatch), st), 'xunet_distill_teacher_step')
    # the second forward sees the same poses, K, cond_mask and parameters: reuse the first one's rays, pose embeddings and
    # weight shadows
    _lib.check(lib.xunet_set_static_conditioning(T.eng.h, 1), 'set_static_conditioning')
    try:
        T.eng.forward(T.flat, train=False)
    finally:
        lib.xunet_set_static_conditioning(T.eng.h, 0)
    _lib.check(lib.xunet_distill_target(T.eng.eps.data_ptr(), w, T.copies, T.table.data_ptr(), T.target.data_ptr(),
                                        T.m.data_ptr(), inp['z'].data_ptr(), T.eng.inp['z'].data_ptr(), B, per,
                                        inp['noise'].data_ptr(), st), 'xunet_distill_target')


def check_teacher(state, teacher: _FrozenTeacher, data) -> None:
    """The ValueErrors of TrainStep(state, data=.., teacher=..): a student is a v / mse state of the teacher's model
    configuration, batch size, image side and device, drawn from a device store without reference quirks; a progressive
    distillation teacher has a grid of even length."""
    if data is None:
        raise ValueError('teacher= distils on batches drawn from a device store: pass data=')
    if state.prediction != 'v' or state.loss != 'mse':
        raise ValueError(f"a distilled student is trained with prediction='v' and loss='mse', this state has "
                         f"prediction={state.prediction!r}, loss={state.loss!r}")
    if state.reference_quirks:
        raise ValueError('teacher= does not take a state with reference_quirks=True')
    if not isinstance(teacher, ConsistencyTeacher) and len(teacher.grid) % 2:
        raise ValueError(f'the teacher grid has odd length {len(teacher.grid)}')
    if teacher.S != state.img_sidelength or teacher.B != state.batch_size:
        raise ValueError(f'the teacher runs B = {teacher.B} at S = {teacher.S}, the student trains B = {state.batch_size} '
                         f'at S = {state.img_sidelength}')
    if teacher.model.config != state.model.config:
        raise ValueError(f'the teacher model {teacher.model.config} differs from the student model {state.model.config}')
    if teacher.device != state.params.flat.device:
        raise ValueError(f'the teacher lives on {teacher.device}, the student on {state.params.flat.device}')
