"""3D consistency score of generated views (3DiM, Watson et al. 2022, section 5): fit a radiance grid to some of the views,
render it at the poses of the others, and score those renders against the held-out views with PSNR / SSIM.  If the views agree
with each other in 3D the grid reproduces the held-out ones; if they disagree about the object's shape it cannot.

    s = consistency_score(views, R, t, K)      # views (V,S,S,3) in [-1, 1], e.g. from Sampler.sample_views; poses per view
    s['mean_psnr'], s['mean_ssim']

The field, its rays and its loss are defined in include/xunet_b200.h (xunet_field_render, xunet_field_loss_grad): a dense
(G, G, G, 4) grid in the cube [-b, b]^3, trilinear, softplus density, sigmoid colour and no view dependence.  Rays use SRN's own
camera model (pixel centre (col + 1/2, row + 1/2), XUNET_RAYS_OPENCV_UV) whatever ray convention the X-UNet checkpoint was
trained with: the convention describes the network, not the cameras.  The fit runs on the GPU (csrc/field.cu): one iteration is
the ray gradient, the finish pass, Adam (xunet_adam_step) and the count, replayed as one CUDA graph; it is deterministic bit for
bit.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .metrics import image_metrics
from .srn_data import mix64

DENSITY_SHIFT = -6.0          # XUNET_FIELD_DENSITY_SHIFT
MIN_GRID, MAX_GRID = 2, 256   # XUNET_FIELD_MIN_GRID, XUNET_FIELD_MAX_GRID
MAX_BOUND = 64.0              # XUNET_FIELD_MAX_BOUND
MAX_SAMPLES = 4096            # XUNET_FIELD_MAX_SAMPLES
MAX_RAYS = 1 << 20            # XUNET_FIELD_MAX_RAYS
FIXED_ONE = 2.0 ** 32         # XUNET_FIELD_FIXED_ONE

# Defaults of fit_field, chosen on the analytic sphere scenes of tests/test_gpu_field.py (40 views at 64^2, G = 64, 8 held out):
# 43.7 dB on the held-out views of the consistent set against 18.3 dB for the inconsistent one.  Stronger total variation
# blurred the consistent fit (1e-3: 35.4 dB, 0.1: 20.7 dB), lr 0.05 / 0.2 and fewer iterations scored lower.  A fit of 40
# views at 128^2 with G = 128 takes 2.1 s on an H100 80GB HBM3 at 700 W (tools/field_cost.py; DESIGN.md section 2).
ITERS = 1500
RAYS = 8192
LR = 0.1
TV = (1e-5, 1e-5)


def draw_rays(seed: int, i: int, rays: int, n_pixels: int) -> np.ndarray:
    """The training pixels xunet_field_loss_grad draws at iteration i (the 1-based Adam count): ray r is pixel
    mix64(seed * 0x9E3779B97F4A7C15 + i * 0xD1B54A32D192ED03 + r) mod n_pixels, an index v S S + row S + col."""
    m = (1 << 64) - 1
    z = (np.uint64((seed * 0x9E3779B97F4A7C15 + i * 0xD1B54A32D192ED03) & m) +
         np.arange(rays, dtype=np.uint64))
    return (mix64(z) % np.uint64(n_pixels)).astype(np.int64)


def default_bound(t) -> float:
    """0.95 min_v |t_v| / sqrt(3): the largest origin-centred cube that no camera centre is inside (SRN's and synthetic.py's
    cameras look at the origin)."""
    return 0.95 * float(np.min(np.linalg.norm(np.asarray(t, np.float64), axis=-1))) / np.sqrt(3.0)


def _dev():
    return torch.device('cuda', torch.cuda.current_device())


def _f32(a, shape_tail: Tuple[int, ...], name: str, dev) -> torch.Tensor:
    x = a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a))
    x = x.to(device=dev, dtype=torch.float32).contiguous()
    if x.ndim != 1 + len(shape_tail) or tuple(x.shape[1:]) != shape_tail:
        raise ValueError(f'{name}: expected shape (V, {", ".join(map(str, shape_tail))}), got {tuple(x.shape)}')
    return x


def _cameras(R, t, K, dev) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    R = _f32(R, (3, 3), 'R', dev)
    t = _f32(t, (3,), 't', dev)
    Kt = K if isinstance(K, torch.Tensor) else torch.as_tensor(np.asarray(K))
    if Kt.ndim == 2:
        Kt = Kt[None].expand(R.shape[0], 3, 3)
    K = _f32(Kt, (3, 3), 'K', dev)
    if not R.shape[0] == t.shape[0] == K.shape[0]:
        raise ValueError(f'R, t and K disagree on the number of views: {R.shape[0]}, {t.shape[0]}, {K.shape[0]}')
    return R, t, K


@dataclass
class Field:
    """A fitted grid: grid (G, G, G, 4) raw values on the device, the cube's bound, the sampling step and near plane, the
    background in [-1, 1], the side S of the views it was fitted to, and loss (iters,), the data loss of each iteration (mean
    squared error of the drawn pixels in [0, 1] units), kept on the device."""
    grid: torch.Tensor
    bound: float
    step: float
    near: float
    background: float
    S: int
    loss: torch.Tensor

    def render(self, R, t, K, S: Optional[int] = None) -> torch.Tensor:
        """(V, S, S, 3) renders in [-1, 1] at the cameras R (V,3,3), t (V,3), K (V,3,3) or (3,3); S defaults to the side of
        the fitted views.  Launched on the current stream; nothing synchronises."""
        dev = self.grid.device
        R, t, K = _cameras(R, t, K, dev)
        S = self.S if S is None else int(S)
        V = R.shape[0]
        out = torch.empty(V, S, S, 3, dtype=torch.float32, device=dev)
        kinv = torch.empty(V, 9, dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(_lib.load().xunet_field_render(self.grid.data_ptr(), self.grid.shape[0], self.bound, R.data_ptr(), t.data_ptr(),
                                                  K.data_ptr(), kinv.data_ptr(), V, S, self.near, self.step, self.background,
                                                  out.data_ptr(), st), 'xunet_field_render')
        return out


def fit_field(views, R, t, K, *, grid: Optional[int] = None, bound: Optional[float] = None, iters: int = ITERS,
              rays: int = RAYS, lr: float = LR, tv: Tuple[float, float] = TV, background: float = 1.0, seed: int = 0,
              step: Optional[float] = None, near: float = 0.0, use_graph: bool = True) -> Field:
    """Fits a radiance grid to views (V, S, S, 3) in [-1, 1] seen from cameras R (V,3,3) cam-to-world, t (V,3), K (V,3,3) or
    (3,3).  grid: G (default S); bound: the cube's half side (default default_bound(t)); step: the sampling step (default half
    the grid spacing, b / (G - 1)); tv: the total-variation weights (density, colour); background in [-1, 1] (SRN: +1, white).
    Each of the `iters` iterations draws `rays` training pixels with replacement and takes one Adam step (lr, b1 = 0.9,
    b2 = 0.99) on the grid, which starts at zero (transparent, grey).  The first iteration runs eagerly, the rest replay it as
    one CUDA graph (use_graph=False: eagerly, with the same bits).  Nothing synchronises."""
    dev = _dev()
    v = views if isinstance(views, torch.Tensor) else torch.as_tensor(np.asarray(views))
    if v.ndim != 4 or v.shape[1] != v.shape[2] or v.shape[3] != 3:
        raise ValueError(f'views: expected shape (V, S, S, 3), got {tuple(v.shape)}')
    v = v.to(device=dev, dtype=torch.float32).contiguous()
    R, t, K = _cameras(R, t, K, dev)
    V, S = v.shape[0], v.shape[1]
    if R.shape[0] != V:
        raise ValueError(f'{V} views but {R.shape[0]} cameras')
    G = S if grid is None else int(grid)
    b = default_bound(t.cpu().numpy()) if bound is None else float(bound)
    dt = b / max(G - 1, 1) if step is None else float(step)
    if iters < 1:
        raise ValueError(f'iters = {iters}, need iters >= 1')
    lib = _lib.load()
    g = torch.zeros(G, G, G, 4, dtype=torch.float32, device=dev)
    m, m2, grad = torch.zeros_like(g), torch.zeros_like(g), torch.empty_like(g)
    acc = torch.zeros(4 * G ** 3 + 1, dtype=torch.int64, device=dev)
    kinv = torch.empty(V, 9, dtype=torch.float32, device=dev)
    count = torch.ones(1, dtype=torch.int64, device=dev)
    loss = torch.zeros(iters, dtype=torch.float32, device=dev)
    tv_d, tv_c = (float(x) for x in tv)

    def one(stream: int) -> None:
        _lib.check(lib.xunet_field_loss_grad(g.data_ptr(), G, b, v.data_ptr(), R.data_ptr(), t.data_ptr(), K.data_ptr(),
                                             kinv.data_ptr(), V, S, near, dt, background, rays,
                                             count.data_ptr(), seed, tv_d, tv_c, acc.data_ptr(), grad.data_ptr(),
                                             loss.data_ptr(), iters, stream), 'xunet_field_loss_grad')
        _lib.check(lib.xunet_adam_step(g.data_ptr(), grad.data_ptr(), m.data_ptr(), m2.data_ptr(), g.numel(), 0,
                                       count.data_ptr(), lr, 0.9, 0.99, 1e-8, 1.0, stream), 'xunet_adam_step')
        count.add_(1)

    one(torch.cuda.current_stream(dev).cuda_stream)
    if iters > 1:
        if use_graph:
            side = torch.cuda.Stream(device=dev)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                one(side.cuda_stream)
            for _ in range(iters - 1):
                graph.replay()
        else:
            for _ in range(iters - 1):
                one(torch.cuda.current_stream(dev).cuda_stream)
    return Field(grid=g, bound=b, step=dt, near=near, background=background, S=S, loss=loss)


def held_out(V: int, every: int) -> list:
    """Indices k < V with k % every == every - 1: the views consistency_score renders instead of fitting."""
    return [k for k in range(V) if k % every == every - 1]


def consistency_score(views, R, t, K, *, every: int = 8, **fit_kw) -> Dict:
    """3D consistency of views (V, S, S, 3) in [-1, 1] seen from R (V,3,3), t (V,3), K (V,3,3) or (3,3): the views k with
    k % every == every - 1 are held out, a grid is fitted to the rest (fit_field, **fit_kw), rendered at the held-out cameras,
    and the renders are scored against the held-out views with image_metrics.  Returns dict(psnr, ssim (lists per held-out
    view), mean_psnr, mean_ssim, held_out (indices), fit_loss (the data loss of the last iteration)); synchronises once.
    Raises ValueError for fewer than 2 views, every < 2, or a split that leaves no view on one side."""
    V = len(views)
    if V < 2:
        raise ValueError(f'need at least 2 views, got {V}')
    if every < 2:
        raise ValueError(f'every = {every}, need every >= 2')
    test = held_out(V, every)
    train = [k for k in range(V) if k not in set(test)]
    if not test or not train:
        raise ValueError(f'{V} views with every = {every} leave {len(train)} to fit and {len(test)} to hold out')
    dev = _dev()
    v = views if isinstance(views, torch.Tensor) else torch.as_tensor(np.asarray(views))
    v = v.to(device=dev, dtype=torch.float32)
    Rc, tc, Kc = _cameras(R, t, K, dev)
    if Rc.shape[0] != V:
        raise ValueError(f'{V} views but {Rc.shape[0]} cameras')
    tr, te = torch.as_tensor(train, device=dev), torch.as_tensor(test, device=dev)
    if 'bound' not in fit_kw or fit_kw['bound'] is None:
        fit_kw['bound'] = default_bound(tc.cpu().numpy())    # from every camera, so no held-out camera is inside the cube
    f = fit_field(v[tr], Rc[tr], tc[tr], Kc[tr], **fit_kw)
    m = image_metrics(f.render(Rc[te], tc[te], Kc[te]), v[te])
    psnr, ssim = m['psnr'].tolist(), m['ssim'].tolist()
    return dict(psnr=psnr, ssim=ssim, mean_psnr=float(np.mean(psnr)), mean_ssim=float(np.mean(ssim)), held_out=test,
                fit_loss=float(f.loss[-1].item()))
