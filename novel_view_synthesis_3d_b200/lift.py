"""Lift one view to a radiance grid by score distillation through the guided X-UNet (DreamFusion's SDS, Poole et al. 2022, on a
view-conditioned model as in Zero-1-to-3 + SJC and Magic123):

    lifter = FieldLifter(model, params, img_sidelength=S, draws=P, w=3.0)
    up, _ = estimate_up(R_all)                         # the world up of the dataset's cameras (or (0, 0, 1))
    res = lifter.lift(x, R1, t1, K, iters=1000, up=up, elevation=(0.0, 60.0))
    res.field.render(R, t, K)                          # (V, S, S, 3) in [-1, 1], as a consistency.Field
    res.field.loss, res.sds                            # per iteration, on the device

The grid (consistency.Field; include/xunet_b200.h defines it) starts at zero.  One iteration, all on the device (csrc/lift.cu,
csrc/field.cu; the header states each entry's arithmetic):
  1. xunet_lift_draw: P cameras on the band of elevations `elevation` against `up` at the source's radius |t1|, looking at the
     origin with zero roll, and P timesteps in t_range, from a hash of (seed, i, p);
  2. xunet_field_render of the P drawn views and the source view;
  3. xunet_lift_noise: z = sqrt(abar) render + sqrt(1 - abar) eps into both halves of the guided batch;
  4. the forward of the 2P rows [cond ; uncond] (cond_mask [1]*P + [0]*P), conditioned on the source view and its camera;
  5. xunet_lift_grad: eps_hat of the guided output (1 + w) o_c - w o_u (converted from v for prediction='v'), the residual
     eps_hat - eps weighted by omega(t) = 1 - abar_t and sds_weight, and the source view's reconstruction gradient weighted by
     recon_weight, as the gradient of a loss w.r.t. the composited colours (the denoiser's Jacobian is not used);
  6. xunet_field_image_grad: that gradient back through the renderer into the grid, plus total variation;
  7. xunet_adam_step on the grid (lr, b1 = 0.9, b2 = 0.99, eps = 1e-8), then the count + 1.
Iteration 1 runs eagerly and the rest replay it as one CUDA graph (use_graph=False: eagerly, the same bits); nothing
synchronises until a result is read.

The lifter runs on the model's inference engine engine(2P, S, False) with input slots of its own, so it never overwrites the
inputs of a Sampler on the same engine; static conditioning stays off, since the target cameras change every iteration.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from .consistency import Field, default_bound
from .diffusion import diffusion_tables
from .pose import LOSS_CHUNK, MAX_T
from .sampling import check_prediction
from .xunet import XUNet, InputSlots

SEED_DOMAIN = 0x6C6966745F736473       # XUNET_LIFT_SEED_DOMAIN
MAX_RESIDUAL = 16.0                    # XUNET_LIFT_MAX_RESIDUAL
MAX_PIXELS = 1 << 20                   # XUNET_FIELD_MAX_RAYS: (P + 1) S^2 at most
MAX_GRAD_L1 = 2.0 ** 23                # XUNET_FIELD_MAX_GRAD_L1

# Defaults, not tuned on a trained checkpoint (none ships with the project): 2 draws per iteration, t away from both ends of
# the schedule, guidance 3 as the sampler, and fit_field's learning rate and total variation.  The elevation band is SRN's
# upper hemisphere.
DRAWS = 2
W = 3.0
T_RANGE = (20, 980)
ITERS = 1000
LR = 0.1
TV = (1e-5, 1e-5)
ELEVATION = (0.0, 60.0)
ADAM = (0.9, 0.99, 1e-8)


def estimate_up(R) -> Tuple[np.ndarray, float]:
    """The world up of zero-roll look-at cameras R (V, 3, 3) cam-to-world, and a residual.  A zero-roll camera's right axis
    (column 0) is perpendicular to up, so up is the least singular vector of the stacked right axes, signed so that it agrees
    with the mean of the cameras' -y axes (image up).  The residual is the RMS of right . up over the cameras: ~0 for zero-roll
    cameras, large (up to ~0.6) for rolled ones.  Needs right axes that span a plane (cameras at two or more azimuths)."""
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    right = R[:, :, 0]
    _, s, vt = np.linalg.svd(right, full_matrices=True)
    up = vt[-1]
    if float(up @ (-R[:, :, 1]).mean(0)) < 0.0:
        up = -up
    return up, float(np.sqrt(np.mean((right @ up) ** 2)))


def grad_unit(sds_weight: float, recon_weight: float) -> float:
    """The unit of the image gradient xunet_lift_grad writes and xunet_field_image_grad scatters: the smallest power of two u
    with (32 sds_weight + 2 recon_weight) / u <= MAX_GRAD_L1, the bound of sum |dC| that keeps the fixed-point sums from
    overflowing (1 when both weights are 0).  In this unit the gradient values are of order 1 rather than 1 / (3 S^2 P), so
    the scatter's quantum of 2^-32 resolves the small per-sample contributions of a nearly empty grid."""
    l1 = 2.0 * MAX_RESIDUAL * float(sds_weight) + 2.0 * float(recon_weight)
    return 1.0 if l1 == 0.0 else 2.0 ** math.ceil(math.log2(l1 / MAX_GRAD_L1))


def elevation_range(t, up) -> Tuple[float, float]:
    """The least and greatest elevation, in degrees, of the camera centres t (V, 3) above the plane perpendicular to up."""
    t = np.asarray(t, np.float64).reshape(-1, 3)
    u = np.asarray(up, np.float64) / np.linalg.norm(up)
    e = np.degrees(np.arcsin(np.clip(t @ u / np.linalg.norm(t, axis=1), -1.0, 1.0)))
    return float(e.min()), float(e.max())


@dataclass
class LiftResult:
    """field: the lifted grid (field.loss (iters,) the source-view reconstruction MSE, in [0, 1] units, of each iteration);
    sds (iters,): the mean squared guided residual |eps_hat - eps|^2 of the P draws of each iteration.  Both on the device."""
    field: Field
    sds: torch.Tensor


class FieldLifter:
    """Lifts a view (S, S, 3) to a radiance grid by score distillation (module docstring).

    draws P: drawn cameras per iteration, so the engine batch is 2P.  w >= 0: the classifier-free guidance weight (w=None,
    a distilled student, is not supported).  prediction: 'eps' or 'v'.  t_range = (t_min, t_max): the integer timesteps drawn,
    0 <= t_min <= t_max <= 999.  grid G: the grid side (default S).  (P + 1) S^2 <= 2^20.  The defaults are not tuned on a
    trained checkpoint.  Raises ValueError for arguments outside these ranges."""

    def __init__(self, model: XUNet, params, img_sidelength: int, *, draws: int = DRAWS, w: Optional[float] = W,
                 prediction: str = 'eps', t_range: Tuple[int, int] = T_RANGE, grid: Optional[int] = None):
        P, S = int(draws), int(img_sidelength)
        if P < 1 or S < 1:
            raise ValueError(f'draws = {P}, img_sidelength = {S}: need both >= 1')
        if (P + 1) * S * S > MAX_PIXELS:
            raise ValueError(f'(draws + 1) S^2 = {(P + 1) * S * S} pixels, need at most {MAX_PIXELS}')
        if w is None:
            raise ValueError('w=None (a distilled student without guidance) is not supported: lifting needs the guided batch')
        w = float(w)
        if not (math.isfinite(w) and w >= 0.0):
            raise ValueError(f'w = {w}: need a finite w >= 0')
        t_min, t_max = (int(v) for v in t_range)
        if not 0 <= t_min <= t_max <= MAX_T:
            raise ValueError(f't_range = ({t_min}, {t_max}): need 0 <= t_min <= t_max <= {MAX_T}')
        G = S if grid is None else int(grid)
        if not 2 <= G <= 256:
            raise ValueError(f'grid = {G}, need 2 <= G <= 256')
        self.prediction = check_prediction(prediction)
        self.P, self.S, self.G, self.w, self.t_min, self.t_max = P, S, G, w, t_min, t_max
        self.model = model
        self.flat = model.flat_from_tree(params, S, 2 * P)
        self.eng = model.engine(2 * P, S, False)
        self.lib = _lib.load()
        dev = self.dev = self.eng.device
        f32 = dict(dtype=torch.float32, device=dev)
        self.slots = InputSlots(2 * P, S, 1, dev)
        self.inp = self.slots.inp[0]
        self.inp['cond_mask'].copy_(torch.cat([torch.ones(P), torch.zeros(P)]))
        sa, sb = diffusion_tables()
        self.sqrt_ac, self.sqrt_1mac = torch.as_tensor(sa).to(dev), torch.as_tensor(sb).to(dev)
        self.cam_R, self.cam_t, self.cam_K = (torch.zeros(P + 1, *s, **f32) for s in ((3, 3), (3,), (3, 3)))
        self.kinv = torch.zeros(P + 1, 9, **f32)
        self.t_draw = torch.zeros(P, dtype=torch.int32, device=dev)
        self.render = torch.zeros(P + 1, S, S, 3, **f32)
        self.eps = torch.zeros(P, S, S, 3, **f32)
        self.dC = torch.zeros(P + 1, S, S, 3, **f32)
        self.partial = torch.zeros((P + 1) * -(-3 * S * S // LOSS_CHUNK), dtype=torch.float64, device=dev)
        self.grid = torch.zeros(G, G, G, 4, **f32)
        self.grad, self.m, self.v = torch.zeros_like(self.grid), torch.zeros_like(self.grid), torch.zeros_like(self.grid)
        self.acc = torch.zeros(4 * G ** 3 + 1, dtype=torch.int64, device=dev)
        self.count = torch.ones(1, dtype=torch.int64, device=dev)

    # ---- the device steps ------------------------------------------------------------------------------------------------
    def _st(self) -> int:
        return torch.cuda.current_stream(self.dev).cuda_stream

    def _iteration(self, a: dict, sds: torch.Tensor, loss: torch.Tensor) -> None:
        lib, P, S, G, i, it = self.lib, self.P, self.S, self.G, self.inp, self.count.data_ptr()
        _lib.check(lib.xunet_lift_draw(P, self.t_min, self.t_max, it, a['seed'], *a['up'], *a['elev'], a['radius'],
                                       i['R2'].data_ptr(), i['t2'].data_ptr(), self.cam_R.data_ptr(), self.cam_t.data_ptr(),
                                       self.t_draw.data_ptr(), self._st()), 'xunet_lift_draw')
        geom = (G, a['bound'])
        tail = (a['near'], a['step'], a['background'])
        _lib.check(lib.xunet_field_render(self.grid.data_ptr(), *geom, self.cam_R.data_ptr(), self.cam_t.data_ptr(),
                                          self.cam_K.data_ptr(), self.kinv.data_ptr(), P + 1, S, *tail, self.render.data_ptr(),
                                          self._st()), 'xunet_field_render')
        _lib.check(lib.xunet_lift_noise(self.render.data_ptr(), self.t_draw.data_ptr(), P, S, it, a['seed'],
                                        self.sqrt_ac.data_ptr(), self.sqrt_1mac.data_ptr(), i['z'].data_ptr(),
                                        i['logsnr'].data_ptr(), self.eps.data_ptr(), self._st()), 'xunet_lift_noise')
        out = self.eng.forward(self.flat, train=False, inputs=(self.slots, 0))
        _lib.check(lib.xunet_lift_grad(out.data_ptr(), i['z'].data_ptr(), self.eps.data_ptr(), self.render.data_ptr(),
                                       i['x'].data_ptr(), self.t_draw.data_ptr(), P, S, self.w, int(self.prediction == 'v'),
                                       a['sds_weight'], a['recon_weight'], a['unit'], self.sqrt_ac.data_ptr(),
                                       self.sqrt_1mac.data_ptr(), it,
                                       self.partial.data_ptr(), self.dC.data_ptr(), sds.data_ptr(), loss.data_ptr(),
                                       loss.shape[0], self._st()), 'xunet_lift_grad')
        _lib.check(lib.xunet_field_image_grad(self.grid.data_ptr(), *geom, self.dC.data_ptr(), a['unit'], self.cam_R.data_ptr(),
                                              self.cam_t.data_ptr(), self.cam_K.data_ptr(), self.kinv.data_ptr(), P + 1, S, *tail,
                                              *a['tv'], self.acc.data_ptr(), self.grad.data_ptr(), self._st()),
                   'xunet_field_image_grad')
        b1, b2, e = ADAM
        _lib.check(lib.xunet_adam_step(self.grid.data_ptr(), self.grad.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                                       self.grid.numel(), 0, it, a['lr'], b1, b2, e, 1.0, self._st()), 'xunet_adam_step')
        self.count.add_(1)

    def _f32(self, a, shape, name) -> torch.Tensor:
        x = a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a))
        if tuple(x.shape) != shape:
            raise ValueError(f'{name}: expected shape {shape}, got {tuple(x.shape)}')
        return x.detach().to(device=self.dev, dtype=torch.float32)

    # ---- public --------------------------------------------------------------------------------------------------------------
    def lift(self, x, R1, t1, K, *, iters: int = ITERS, up=(0.0, 0.0, 1.0), elevation: Tuple[float, float] = ELEVATION,
             lr: float = LR, tv: Tuple[float, float] = TV, sds_weight: float = 1.0, recon_weight: float = 1.0,
             background: float = 1.0, seed: int = 0, use_graph: bool = True) -> LiftResult:
        """Lifts x (S,S,3) in [-1, 1], seen from R1 (3,3) cam-to-world, t1 (3,) with intrinsics K (3,3), to a fresh grid.
        up: the world up of the drawn cameras (estimate_up); elevation = (lo, hi) in degrees within [-90, 90]: the band of
        camera elevations against up, at radius |t1|; the cube's bound is default_bound(t1) and the step half a grid spacing,
        as fit_field.  lr: Adam's learning rate; tv = (density, colour) total-variation weights; sds_weight and recon_weight
        scale the distillation and source-reconstruction terms (finite, >= 0); background in [-1, 1] (SRN: +1, white).  Each of
        the `iters` iterations draws afresh from (seed, iteration); the first runs eagerly and the rest replay it as one CUDA
        graph (use_graph=False: eagerly, the same bits).  Nothing synchronises, except that a t1 given as a device tensor is
        read back to the host: its length places the drawn cameras and sizes the cube."""
        S, P = self.S, self.P
        iters = int(iters)
        if iters < 1:
            raise ValueError(f'iters = {iters}, need iters >= 1')
        x = self._f32(x, (S, S, 3), 'x')
        R1 = self._f32(R1, (3, 3), 'R1')
        t1h = (t1.detach().cpu() if isinstance(t1, torch.Tensor) else torch.as_tensor(np.asarray(t1))).to(torch.float32)
        if tuple(t1h.shape) != (3,):
            raise ValueError(f't1: expected shape (3,), got {tuple(t1h.shape)}')
        t1 = t1h.to(self.dev)
        K = self._f32(K, (3, 3), 'K')
        upv = np.asarray(up, np.float64)
        if upv.shape != (3,) or not np.all(np.isfinite(upv)) or not np.linalg.norm(upv) > 0.0:
            raise ValueError(f'up = {up!r}: need a finite nonzero 3-vector')
        lo, hi = (float(e) for e in elevation)
        if not -90.0 <= lo <= hi <= 90.0:
            raise ValueError(f'elevation = ({lo}, {hi}): need -90 <= lo <= hi <= 90 degrees')
        radius = float(np.linalg.norm(t1h.double().numpy()))
        if not radius > 0.0:
            raise ValueError('t1 = 0: the drawn cameras need a source camera away from the origin')
        lr, sw, rw = float(lr), float(sds_weight), float(recon_weight)
        if not (math.isfinite(lr) and lr >= 0.0):
            raise ValueError(f'lr = {lr}: need a finite lr >= 0')
        if not (math.isfinite(sw) and sw >= 0.0):
            raise ValueError(f'sds_weight = {sw}: need a finite weight >= 0')
        if not (math.isfinite(rw) and rw >= 0.0):
            raise ValueError(f'recon_weight = {rw}: need a finite weight >= 0')
        tv_d, tv_c = (float(v) for v in tv)
        if not (math.isfinite(tv_d) and math.isfinite(tv_c) and tv_d >= 0.0 and tv_c >= 0.0):
            raise ValueError(f'tv = {tv!r}: need finite weights >= 0')
        background = float(background)
        if not math.isfinite(background):
            raise ValueError(f'background = {background}: need a finite value')
        b = default_bound(t1h.numpy()[None])
        a = dict(seed=int(seed) & 0xFFFFFFFFFFFFFFFF, up=tuple(upv / np.linalg.norm(upv)),
                 elev=(math.radians(lo), math.radians(hi)), radius=radius, bound=b, step=b / (self.G - 1), near=0.0,
                 background=background, sds_weight=sw, recon_weight=rw, unit=grad_unit(sw, rw), lr=lr, tv=(tv_d, tv_c))
        self._a = a                     # the arguments of the last lift, which its iterations read
        i = self.inp
        i['x'].copy_(x.expand_as(i['x']))
        i['R1'].copy_(R1.expand_as(i['R1']))
        i['t1'].copy_(t1.expand_as(i['t1']))
        i['K'].copy_(K.expand_as(i['K']))
        self.cam_R[P].copy_(R1)
        self.cam_t[P].copy_(t1)
        self.cam_K.copy_(K.expand_as(self.cam_K))
        self.grid.zero_()
        self.m.zero_()
        self.v.zero_()
        self.count.fill_(1)
        sds = torch.zeros(iters, dtype=torch.float32, device=self.dev)
        loss = torch.zeros(iters, dtype=torch.float32, device=self.dev)
        self._iteration(a, sds, loss)
        if iters > 1:
            if use_graph:
                side = torch.cuda.Stream(device=self.dev)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=side):
                    self._iteration(a, sds, loss)
                for _ in range(iters - 1):
                    graph.replay()
            else:
                for _ in range(iters - 1):
                    self._iteration(a, sds, loss)
        field = Field(grid=self.grid.clone(), bound=b, step=a['step'], near=0.0, background=background, S=S, loss=loss)
        return LiftResult(field=field, sds=sds)
