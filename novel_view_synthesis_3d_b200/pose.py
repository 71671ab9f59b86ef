"""Estimate the camera of a view by descending the denoising loss of a view-conditioned model (ID-Pose, iFusion, 2023):

    est = PoseEstimator(model, params, img_sidelength=S, hypotheses=H, draws=P)
    res = est.estimate(x, R1, t1, K, y, iters=200)     # x at the known camera (R1, t1), K; y the view whose camera is wanted
    res.R_best, res.t_best                              # the hypothesis with the lowest evaluation loss
    rotation_error_deg(res.R_best, R_true)

H pose hypotheses are fitted side by side; each sees P noise draws per iteration, so the engine batch is B = H P, and row
b = h P + p is hypothesis h with draw p.  All hypotheses share draw p (common random numbers: the loss differences between
hypotheses come from the pose alone).  One iteration, all on the device (csrc/pose_fit.cu; include/xunet_b200.h states each
entry's arithmetic):
  1. xunet_pose_draw: t_p uniform in [t_min, t_max] and eps_p from a seed mixed from (seed, i, p); z_b, logsnr_b into the input
     slots, and the regression target (eps_p, or v for prediction='v') of each draw;
  2. the forward (train=0) with cond_mask 1;
  3. xunet_pose_loss: L_h = (1/P) sum_p mean (out_b - target_p)^2 into row i-1 of the loss history, and its seed dL/d(out);
  4. xunet_backward_vjp_inputs for dL/dR2 and dL/dt2;
  5. xunet_pose_tangent: the gradient in the tangent coordinates (omega, delta) of R' = exp([omega]x) R, t' = exp([omega]x) t +
     delta, a rotation about the world origin (the object's centre in SRN, whose cameras lie on a sphere and look at it), plus
     a translation with translate=True;
  6. xunet_adam_step on a zero step buffer (lr, b1 = 0.9, b2 = 0.999, eps = 1e-8);
  7. xunet_pose_retract: R <- exp([omega]x) R, t <- exp([omega]x) t + delta on fp64 master poses, the fp32 poses into the
     slots;
  8. the count + 1.
Iteration 1 runs eagerly and the rest replay it as one CUDA graph; nothing synchronises until a result is read.

The estimator runs on the model's training engine engine(H P, S, True) with input slots of its own, the way TrainStep does:
a vjp taken on that engine must be finished before an estimate, whose forwards replace its activations.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Optional, Tuple, Union

import numpy as np
import torch

from . import _lib
from .diffusion import diffusion_tables
from .sampling import check_prediction
from .xunet import XUNet, InputSlots

MAX_T = 999                  # XUNET_POSE_MAX_T
LOSS_CHUNK = 4096            # XUNET_POSE_LOSS_CHUNK
SMALL_ANGLE2 = 1e-6          # XUNET_POSE_SMALL_ANGLE2
EVAL_SEED = 0x3C6EF372FE94F82B   # the draws of score(): the same for every hypothesis and every estimate
ADAM = (0.9, 0.999, 1e-8)    # b1, b2, eps

# Defaults, not tuned on a trained checkpoint (none ships with the project): 8 starts spread over the sphere, 2 draws each,
# 200 iterations of Adam at 0.01 rad (at most ~2 rad of travel), t away from both ends of the schedule, 8 evaluation draws.
HYPOTHESES = 8
DRAWS = 2
ITERS = 200
LR = 0.01
T_RANGE = (100, 900)


def _np64(a) -> np.ndarray:
    return (a.detach().cpu().double().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, dtype=np.float64))


def fibonacci_sphere(n: int) -> np.ndarray:
    """(n, 3) unit vectors of the Fibonacci lattice: z_k = 1 - (2k + 1) / n, azimuth k pi (3 - sqrt 5)."""
    k = np.arange(n, dtype=np.float64)
    z = 1.0 - (2.0 * k + 1.0) / n
    r = np.sqrt(np.maximum(0.0, 1.0 - z * z))
    phi = k * math.pi * (3.0 - math.sqrt(5.0))
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], -1)


def rotation_between(a, b) -> np.ndarray:
    """The smallest rotation (3, 3) taking the unit vector a to the unit vector b.  Antipodal b = -a: the half turn about the
    axis a x e, e the basis vector least aligned with a."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    c = float(a @ b)
    if 1.0 + c < 1e-8:
        e = np.eye(3)[int(np.argmin(np.abs(a)))]
        n = np.cross(a, e)
        n /= np.linalg.norm(n)
        return 2.0 * np.outer(n, n) - np.eye(3)
    v = np.cross(a, b)
    V = np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])
    return np.eye(3) + V + V @ V / (1.0 + c)


def sphere_init(R1, t1, H: int) -> Tuple[np.ndarray, np.ndarray]:
    """H starting cameras (R (H,3,3), t (H,3), fp64) on the sphere of radius |t1|: hypothesis h is camera 1 rotated about the
    origin by the smallest rotation taking t1 / |t1| to point h of the Fibonacci lattice.  The roll comes from camera 1 (no
    world "up" is assumed), and a camera 1 that looks at the origin gives hypotheses that do too."""
    R1, t1 = _np64(R1).reshape(3, 3), _np64(t1).reshape(3)
    r = float(np.linalg.norm(t1))
    if not r > 0.0:
        raise ValueError('t1 = 0: the sphere start needs a camera away from the origin')
    Q = np.stack([rotation_between(t1 / r, u) for u in fibonacci_sphere(H)])
    return Q @ R1, Q @ t1


def rotation_error_deg(Ra, Rb) -> np.ndarray:
    """The geodesic angle, in degrees, of Ra Rb^T for rotations (..., 3, 3) (numpy or torch): atan2(|vee(M - M^T)| / 2,
    (tr M - 1) / 2), accurate near 0 and 180 degrees."""
    Ra, Rb = _np64(Ra), _np64(Rb)
    M = Ra @ np.swapaxes(Rb, -1, -2)
    s = 0.5 * np.linalg.norm(np.stack([M[..., 2, 1] - M[..., 1, 2], M[..., 0, 2] - M[..., 2, 0], M[..., 1, 0] - M[..., 0, 1]], -1),
                             axis=-1)
    c = 0.5 * (M[..., 0, 0] + M[..., 1, 1] + M[..., 2, 2] - 1.0)
    return np.degrees(np.arctan2(s, c))


@dataclass
class PoseResult:
    """R (H,3,3), t (H,3): the final fp64 poses of the hypotheses; score (H,) fp64: their evaluation loss (PoseEstimator.score);
    loss (iters, H) fp32: the training loss L_h of every iteration.  All on the device; best and the *_best fields read them."""
    R: torch.Tensor
    t: torch.Tensor
    score: torch.Tensor
    loss: torch.Tensor

    @property
    def best(self) -> int:
        return int(torch.argmin(self.score))

    @property
    def R_best(self) -> torch.Tensor:
        return self.R[self.best]

    @property
    def t_best(self) -> torch.Tensor:
        return self.t[self.best]


class PoseEstimator:
    """Estimates the camera of a target view y from a conditioning view x at a known camera (module docstring).

    hypotheses H, draws P: the engine batch is H P.  prediction: what the network predicts, 'eps' or 'v'.  t_range =
    (t_min, t_max): the integer timesteps drawn, 0 <= t_min <= t_max <= 999.  lr: Adam's learning rate in radians (and scene
    units for the translation), finite and >= 0.  translate=False fits the rotation about the origin only (3 DoF, exact for
    SRN's cameras); True fits a translation too (6 DoF, for refining general poses).  eval_draws E (a multiple of P, default
    4 P): the draws score() averages, with timesteps stratified over t_range.  The defaults are not tuned on a trained
    checkpoint.  Raises ValueError for arguments outside these ranges."""

    def __init__(self, model: XUNet, params, img_sidelength: int, *, hypotheses: int = HYPOTHESES, draws: int = DRAWS,
                 prediction: str = 'eps', t_range: Tuple[int, int] = T_RANGE, lr: float = LR, translate: bool = False,
                 eval_draws: Optional[int] = None):
        H, P, S = int(hypotheses), int(draws), int(img_sidelength)
        if H < 1 or P < 1:
            raise ValueError(f'hypotheses = {H}, draws = {P}: need both >= 1')
        if S < 1:
            raise ValueError(f'img_sidelength = {S}, need S >= 1')
        t_min, t_max = (int(v) for v in t_range)
        if not 0 <= t_min <= t_max <= MAX_T:
            raise ValueError(f't_range = ({t_min}, {t_max}): need 0 <= t_min <= t_max <= {MAX_T}')
        lr = float(lr)
        if not (math.isfinite(lr) and lr >= 0.0):
            raise ValueError(f'lr = {lr}: need a finite lr >= 0')
        self.prediction = check_prediction(prediction)
        E = 4 * P if eval_draws is None else int(eval_draws)
        if E < P or E % P:
            raise ValueError(f'eval_draws = {E}: need a positive multiple of draws = {P}')
        self.H, self.P, self.S, self.E = H, P, S, E
        self.t_min, self.t_max, self.lr, self.translate = t_min, t_max, lr, bool(translate)
        self.D = 6 if self.translate else 3
        self.model = model
        self.flat = model.flat_from_tree(params, S)
        self.eng = model.engine(H * P, S, True)
        self.lib = _lib.load()
        dev = self.dev = self.eng.device
        B, D = H * P, self.D
        f32, f64 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.float64, device=dev)
        self.slots = InputSlots(B, S, 1, dev)            # cond_mask 1 for every row
        self.inp = self.slots.inp[0]
        sa, sb = diffusion_tables()
        self.sqrt_ac, self.sqrt_1mac = torch.as_tensor(sa).to(dev), torch.as_tensor(sb).to(dev)
        self.y = torch.zeros(S, S, 3, **f32)
        self.target = torch.zeros(P, S, S, 3, **f32)
        self.d_eps = torch.zeros(B, S, S, 3, **f32)
        self.partial = torch.zeros(B * -(-3 * S * S // LOSS_CHUNK), **f64)
        self.d_rays = torch.zeros(B, 2, S, S, 6, **f32)
        self.dR = torch.zeros(B, 3, 3, **f32)
        self.dt = torch.zeros(B, 3, **f32)
        self.R = torch.zeros(H, 3, 3, **f64)             # fp64 master poses
        self.t = torch.zeros(H, 3, **f64)
        self.step = torch.zeros(H, D, **f32)             # Adam's "parameters": zero on entry, the update after
        self.grad = torch.zeros(H, D, **f32)
        self.m, self.v = torch.zeros(H, D, **f32), torch.zeros(H, D, **f32)
        self.count = torch.ones(1, dtype=torch.int64, device=dev)
        self.eval_iters = torch.arange(1, E // P + 1, dtype=torch.int64, device=dev)
        self._grads = _lib.XunetInputGrads(d_rays=self.d_rays.data_ptr(), dR2=self.dR.data_ptr(), dt2=self.dt.data_ptr())

    # ---- the device steps ------------------------------------------------------------------------------------------------
    def _st(self) -> int:
        return torch.cuda.current_stream(self.dev).cuda_stream

    def _draw(self, iter_ptr: int, seed: int, strata: int) -> None:
        i = self.inp
        _lib.check(self.lib.xunet_pose_draw(self.y.data_ptr(), self.H, self.P, self.S, self.t_min, self.t_max, strata, iter_ptr,
                                            seed & 0xFFFFFFFFFFFFFFFF, self.sqrt_ac.data_ptr(), self.sqrt_1mac.data_ptr(),
                                            int(self.prediction == 'v'), i['z'].data_ptr(), i['logsnr'].data_ptr(),
                                            self.target.data_ptr(), None, self._st()), 'xunet_pose_draw')

    def _forward_loss(self, iter_ptr: int, loss: torch.Tensor) -> None:
        out = self.eng.forward(self.flat, train=False, inputs=(self.slots, 0))
        _lib.check(self.lib.xunet_pose_loss(out.data_ptr(), self.target.data_ptr(), self.H, self.P, self.S, iter_ptr,
                                            self.partial.data_ptr(), self.d_eps.data_ptr(), loss.data_ptr(), loss.shape[0],
                                            self._st()), 'xunet_pose_loss')

    def _tangent(self) -> None:
        e = self.eng
        _lib.check(self.lib.xunet_backward_vjp_inputs(e.h, self.flat.data_ptr(), C.byref(self.slots.cbatch[0]),
                                                      self.d_eps.data_ptr(), e.seed.data_ptr(), e.ws.data_ptr(),
                                                      e.grads.data_ptr(), 0, C.byref(self._grads), self._st()),
                   'xunet_backward_vjp_inputs')
        _lib.check(self.lib.xunet_pose_tangent(self.dR.data_ptr(), self.dt.data_ptr(), self.H, self.P, self.R.data_ptr(),
                                               self.t.data_ptr(), int(self.translate), self.grad.data_ptr(), self._st()),
                   'xunet_pose_tangent')

    def _retract(self) -> None:
        _lib.check(self.lib.xunet_pose_retract(self.step.data_ptr(), self.H, self.P, int(self.translate), self.R.data_ptr(),
                                               self.t.data_ptr(), self.inp['R2'].data_ptr(), self.inp['t2'].data_ptr(),
                                               self._st()), 'xunet_pose_retract')

    def _iteration(self, seed: int, loss: torch.Tensor) -> None:
        self._draw(self.count.data_ptr(), seed, 0)
        self._forward_loss(self.count.data_ptr(), loss)
        self._tangent()
        b1, b2, eps = ADAM
        _lib.check(self.lib.xunet_adam_step(self.step.data_ptr(), self.grad.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                                            self.step.numel(), 0, self.count.data_ptr(), self.lr, b1, b2, eps, 1.0, self._st()),
                   'xunet_adam_step')
        self._retract()
        self.count.add_(1)

    # ---- inputs ----------------------------------------------------------------------------------------------------------
    def _f32(self, a, shape, name) -> torch.Tensor:
        x = a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a))
        if tuple(x.shape) != shape:
            raise ValueError(f'{name}: expected shape {shape}, got {tuple(x.shape)}')
        return x.detach().to(device=self.dev, dtype=torch.float32)

    def _poses(self, R, t) -> Tuple[torch.Tensor, torch.Tensor]:
        H = self.H
        R = R if isinstance(R, torch.Tensor) else torch.as_tensor(np.asarray(R))
        t = t if isinstance(t, torch.Tensor) else torch.as_tensor(np.asarray(t))
        if tuple(R.shape) != (H, 3, 3) or tuple(t.shape) != (H, 3):
            raise ValueError(f'poses: expected R ({H}, 3, 3) and t ({H}, 3) for {H} hypotheses, got {tuple(R.shape)} and '
                             f'{tuple(t.shape)}')
        return R.detach().to(device=self.dev, dtype=torch.float64), t.detach().to(device=self.dev, dtype=torch.float64)

    def _set_poses(self, R, t) -> None:
        R, t = self._poses(R, t)
        self.R.copy_(R)
        self.t.copy_(t)
        self.step.zero_()
        self._retract()                  # a zero step: the rows receive the poses as they are

    # ---- public --------------------------------------------------------------------------------------------------------------
    def estimate(self, x, R1, t1, K, y, *, iters: int = ITERS, init: Union[str, Tuple] = 'sphere', seed: int = 0,
                 use_graph: bool = True, rays=None) -> PoseResult:
        """Estimates the camera of y (S,S,3) in [-1, 1] given x (S,S,3) seen from R1 (3,3) cam-to-world, t1 (3,) with
        intrinsics K (3,3).  init='sphere': sphere_init(R1, t1, H); init=(R (H,3,3), t (H,3)): start from given poses
        (refinement).  Each of the `iters` iterations draws afresh from (seed, iteration); iteration 1 runs eagerly and the rest
        replay it as one CUDA graph (use_graph=False: eagerly, the same bits).  The final poses are then scored (score()).
        Explicit rays are refused: the camera gradient needs rays generated from R, t, K.  Nothing synchronises."""
        if rays is not None:
            raise ValueError('explicit rays: the camera gradient needs rays generated from R, t, K')
        S, H = self.S, self.H
        iters = int(iters)
        if iters < 1:
            raise ValueError(f'iters = {iters}, need iters >= 1')
        x = self._f32(x, (S, S, 3), 'x')
        y = self._f32(y, (S, S, 3), 'y')
        R1 = self._f32(R1, (3, 3), 'R1')
        t1 = self._f32(t1, (3,), 't1')
        K = self._f32(K, (3, 3), 'K')
        if isinstance(init, str):
            if init != 'sphere':
                raise ValueError(f"init must be 'sphere' or a pair (R, t), got {init!r}")
            init = sphere_init(R1.cpu(), t1.cpu(), H)
        R0, t0 = init
        self._poses(R0, t0)              # shapes checked before anything is written
        i = self.inp
        i['x'].copy_(x.expand_as(i['x']))
        i['R1'].copy_(R1.expand_as(i['R1']))
        i['t1'].copy_(t1.expand_as(i['t1']))
        i['K'].copy_(K.expand_as(i['K']))
        self.y.copy_(y)
        self.m.zero_()
        self.v.zero_()
        self.count.fill_(1)
        self._set_poses(R0, t0)
        loss = torch.zeros(iters, H, dtype=torch.float32, device=self.dev)
        self._iteration(int(seed), loss)
        if iters > 1:
            if use_graph:
                side = torch.cuda.Stream(device=self.dev)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=side):
                    self._iteration(int(seed), loss)
                for _ in range(iters - 1):
                    graph.replay()
            else:
                for _ in range(iters - 1):
                    self._iteration(int(seed), loss)
        R, t = self.R.clone(), self.t.clone()
        return PoseResult(R=R, t=t, score=self._evaluate(False)[0], loss=loss)

    def _evaluate(self, grad: bool):
        """The evaluation loss of the poses in the rows (and, grad=True, its tangent gradient (H, D))."""
        n = self.E // self.P
        hist = torch.zeros(n, self.H, dtype=torch.float32, device=self.dev)
        g = torch.zeros(self.H, self.D, dtype=torch.float64, device=self.dev) if grad else None
        for c in range(n):
            ptr = self.eval_iters[c:c + 1].data_ptr()
            self._draw(ptr, EVAL_SEED, self.E)
            self._forward_loss(ptr, hist)
            if grad:
                self._tangent()
                g += self.grad.double()
        return hist.double().mean(0), (None if g is None else g / n)

    def score(self, R, t, *, grad: bool = False):
        """The evaluation loss (H,) fp64 of poses R (H,3,3), t (H,3) for the views of the last estimate(): the mean of L_h over
        the E evaluation draws, timesteps stratified over t_range and noise from a fixed seed, the same for every hypothesis
        and independent of the training draws; forward passes only.  grad=True also returns its gradient (H, D) in the tangent
        coordinates (omega, delta) of each pose, from the same kernels an iteration uses.  The estimator's master poses become
        R, t."""
        self._set_poses(R, t)
        s, g = self._evaluate(grad)
        return (s, g) if grad else s
