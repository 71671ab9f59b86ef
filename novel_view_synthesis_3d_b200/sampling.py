"""DDPM ancestral sampler with classifier-free guidance (reference sampling.py:16-53, 73-76, 119-151) on the CUDA path.

Reference behaviour (steps=1000, w=3): per step two model evaluations (cond_mask=1 / 0) -- here ONE forward of a 2B batch
[cond ; uncond] -- eps=(1+w)eps_c-w eps_u, x0=clip(predict_start_from_noise), posterior mean/variance, z<-mean+sigma*N(0,1)
(no noise at t=0), and the log-SNR fed to the network lags one step and starts at -20 (sampling.py:126,151).
`steps<1000` re-spaces the schedule (strided alpha-bar), which is what the 256-step metric uses.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from .xunet import XUNet, BATCH_KEYS


def cosine_beta_schedule(timesteps, s=0.008):
    """sampling.py:16-26 (float64)."""
    steps = timesteps + 1
    x = np.linspace(0, timesteps, steps, dtype=np.float64)
    ac = np.cos(((x / timesteps) + s) / (1 + s) * np.pi * 0.5) ** 2
    ac = ac / ac[0]
    betas = 1 - (ac[1:] / ac[:-1])
    return np.clip(betas, 0, 0.9999)


def logsnr_schedule_cosine(t, *, logsnr_min=-20., logsnr_max=20.):
    """sampling.py:73-76."""
    b = np.arctan(np.exp(-.5 * logsnr_max))
    a = np.arctan(np.exp(-.5 * logsnr_min)) - b
    return -2. * np.log(np.tan(a * t + b))


class Schedule:
    """The tables of sampling.py:28-41, optionally re-spaced to `steps` < T timesteps."""

    def __init__(self, steps: int = 1000, T: int = 1000):
        betas_full = cosine_beta_schedule(T)
        ac_full = np.cumprod(1. - betas_full, axis=0)
        if steps >= T:
            self.timesteps = np.arange(T)
            ac = ac_full
        else:
            self.timesteps = np.unique(np.round(np.linspace(0, T - 1, steps)).astype(int))
            ac = ac_full[self.timesteps]
        ac_prev = np.pad(ac[:-1], (1, 0), 'constant', constant_values=(1))
        betas = 1. - ac / ac_prev
        alphas = 1. - betas
        self.betas, self.alphas_cumprod, self.alphas_cumprod_prev = betas, ac, ac_prev
        self.sqrt_recip_alphas_cumprod = np.sqrt(1. / ac)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1. / ac - 1)
        self.posterior_variance = betas * (1. - ac_prev) / (1. - ac)
        self.posterior_log_variance_clipped = np.log(self.posterior_variance.clip(min=1e-20))
        self.posterior_mean_coef1 = betas * np.sqrt(ac_prev) / (1. - ac)
        self.posterior_mean_coef2 = (1. - ac_prev) * np.sqrt(alphas) / (1. - ac)
        self.T = T

    def __len__(self):
        return len(self.timesteps)


class Sampler:
    def __init__(self, model: XUNet, params, batch_size: int, img_sidelength: int, *, steps: int = 1000, w: float = 3.0,
                 use_graph: bool = True):
        self.model, self.B, self.S, self.w = model, batch_size, img_sidelength, float(w)
        self.sched = Schedule(steps)
        self.eng = model.engine(2 * batch_size, img_sidelength, False)
        self.flat = model.flat_from_tree(params, img_sidelength, 2 * batch_size)
        self.lib = _lib.load()
        self.dev = self.eng.device
        self.z = torch.zeros(batch_size, img_sidelength, img_sidelength, 3, dtype=torch.float32, device=self.dev)
        self.use_graph = use_graph
        self.graph = None
        self._tab = None
        self._pos = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self._seed_base = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.graph_step = None

    def _forward(self, first: bool):
        # poses / params are constant over the loop: only the first step computes rays, posenc, pose convs, weight shadows
        if first:
            self.lib.xunet_set_static_conditioning(self.eng.h, 0)
            self.eng.forward(self.flat, train=False)
            self.lib.xunet_set_static_conditioning(self.eng.h, 1)
            return
        if not self.use_graph:
            self.eng.forward(self.flat, train=False)
            return
        if self.graph is None:
            torch.cuda.synchronize(self.dev)
            st = torch.cuda.Stream(device=self.dev)
            with torch.cuda.stream(st):
                self.eng.forward(self.flat, train=False)
                st.synchronize()
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph, stream=st):
                    self.eng.forward(self.flat, train=False)
            torch.cuda.synchronize(self.dev)
        self.graph.replay()

    def capture(self, batch: dict) -> None:
        """Builds the static-conditioning state and the per-step CUDA graph without running the loop (benchmarks warm up
        with this instead of a full `steps`-long sample)."""
        if self.use_graph:
            self.sample(batch, seed=0, _max_steps=3)
            return
        saved = self.sched
        try:
            self.sched = Schedule(3)
            self.sample(batch, seed=0)
        finally:
            self.sched = saved

    def sample(self, batch: dict, *, seed: int = 0, z_init=None, noises=None, _max_steps=None) -> torch.Tensor:
        """Generates the target view for each (source image, pose pair) in `batch` (keys as data_loader.py:102-113).
        z_init / noises (list per step, index = step position high->low) make the run reproducible against the oracle."""
        B, S, e = self.B, self.S, self.eng
        # only the source image, the two poses and K condition the sampler; z / logsnr are produced by the loop itself
        # (the reference overwrites both before the first step, sampling.py:125-126)
        src = dict(batch)
        src.setdefault('z', np.zeros((B, S, S, 3), np.float32))
        src.setdefault('logsnr', np.zeros((B,), np.float32))
        dup = {k: np.concatenate([np.asarray(src[k], dtype=np.float32)] * 2, axis=0) for k in BATCH_KEYS}
        mask = np.concatenate([np.ones(B, np.float32), np.zeros(B, np.float32)])
        e.load_inputs(dup, cond_mask=mask)
        if z_init is None:
            g = torch.Generator(device=self.dev).manual_seed(seed)
            self.z.copy_(torch.randn(self.z.shape, generator=g, device=self.dev))       # sampling.py:125
        else:
            self.z.copy_(torch.as_tensor(np.asarray(z_init), dtype=torch.float32).to(self.dev))
        logsnr = -20.0                                                                  # sampling.py:126
        sc = self.sched
        n = B * S * S * 3
        if noises is None and self.use_graph:
            return self._sample_device_schedule(seed, _max_steps)
        try:
            for i in range(len(sc) - 1, -1, -1):
                first = i == len(sc) - 1
                e.inp['z'][:B].copy_(self.z)
                e.inp['z'][B:].copy_(self.z)
                e.inp['logsnr'].fill_(float(logsnr))
                self._forward(first)
                sigma = 0.0 if i == 0 else float(np.exp(0.5 * sc.posterior_log_variance_clipped[i]))   # sampling.py:142-148
                noise_ptr = None
                if noises is not None:
                    nz = torch.as_tensor(np.asarray(noises[len(sc) - 1 - i]), dtype=torch.float32).to(self.dev).contiguous()
                    noise_ptr = nz.data_ptr()
                st = torch.cuda.current_stream(self.dev).cuda_stream
                _lib.check(self.lib.xunet_sampler_update(e.eps.data_ptr(), self.z.data_ptr(), noise_ptr, self.z.data_ptr(), n,
                                                         self.w, float(sc.sqrt_recip_alphas_cumprod[i]),
                                                         float(sc.sqrt_recipm1_alphas_cumprod[i]),
                                                         float(sc.posterior_mean_coef1[i]), float(sc.posterior_mean_coef2[i]),
                                                         sigma, (seed * 1000003 + i) & 0xFFFFFFFFFFFFFFFF, st), 'sampler_update')
                logsnr = logsnr_schedule_cosine(sc.timesteps[i] / 1000.0)                   # sampling.py:151
        finally:
            # a failure mid-loop must not leave the shared engine reusing stale pose embeddings / weight shadows
            self.lib.xunet_set_static_conditioning(e.h, 0)
        return self.z.clone()


    # ---- device-side schedule: ONE graph per step (forward + ancestral update + counter), nothing else in the loop ------
    def _table(self) -> torch.Tensor:
        sc = self.sched
        key = (len(sc), int(sc.timesteps[-1]))
        if self._tab is None or self._tab[0] != key:
            rows = []
            for i in range(len(sc) - 1, -1, -1):           # loop position k = len-1-i
                sigma = 0.0 if i == 0 else float(np.exp(0.5 * sc.posterior_log_variance_clipped[i]))   # sampling.py:142-148
                rows.append([sc.sqrt_recip_alphas_cumprod[i], sc.sqrt_recipm1_alphas_cumprod[i], sc.posterior_mean_coef1[i],
                             sc.posterior_mean_coef2[i], sigma, logsnr_schedule_cosine(sc.timesteps[i] / 1000.0), 0.0, 0.0])
            self._tab = (key, torch.as_tensor(np.asarray(rows, dtype=np.float64), dtype=torch.float32).to(self.dev).contiguous())
            self.graph_step = None          # the table pointer is baked into the captured graph
        return self._tab[1]

    def _device_step(self):
        e = self.eng
        st = torch.cuda.current_stream(self.dev).cuda_stream
        _lib.check(self.lib.xunet_sampler_step_table(e.eps.data_ptr(), self.z.data_ptr(), self.B * self.S * self.S * 3, self.w,
                                                     self._table().data_ptr(), self._pos.data_ptr(), self._seed_base.data_ptr(),
                                                     e.inp['z'].data_ptr(), e.inp['logsnr'].data_ptr(), 2 * self.B, st),
                   'sampler_step_table')
        self._pos.add_(1)

    def _sample_device_schedule(self, seed: int, max_steps: Optional[int] = None) -> torch.Tensor:
        """z, the forward's z / log-SNR inputs, the schedule position, the noise seed and the coefficient table all live on
        the device; step 0 runs eagerly (it builds rays, pose embeddings and weight shadows), steps 1.. replay one graph each."""
        B, e = self.B, self.eng
        steps = len(self.sched) if max_steps is None else min(max_steps, len(self.sched))
        self._seed_base.fill_((seed * 1000003 + len(self.sched) - 1) & 0x7FFFFFFFFFFFFFFF)    # same per-step seeds as the host loop
        self._table()
        self._pos.zero_()
        e.inp['z'][:B].copy_(self.z)
        e.inp['z'][B:].copy_(self.z)
        e.inp['logsnr'].fill_(-20.0)                                                    # sampling.py:126
        try:
            self.lib.xunet_set_static_conditioning(e.h, 0)
            e.forward(self.flat, train=False)
            self.lib.xunet_set_static_conditioning(e.h, 1)
            self._device_step()
            if steps > 1 and self.graph_step is None:
                torch.cuda.synchronize(self.dev)
                pos0 = self._pos.clone()
                st = torch.cuda.Stream(device=self.dev)
                with torch.cuda.stream(st):
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=st):
                        e.forward(self.flat, train=False)
                        self._device_step()
                torch.cuda.synchronize(self.dev)
                self._pos.copy_(pos0)
                self.graph_step = g
            for _ in range(steps - 1):
                self.graph_step.replay()
        finally:
            self.lib.xunet_set_static_conditioning(e.h, 0)
        return self.z.clone()

    # ---- stochastic conditioning (3DiM, Watson et al. 2022, section 3.2; the reference implements only k = 1) ---------
    def sample_views(self, views, poses, K, target_poses, *, seed: int = 0, condition_on_generated: bool = True,
                     return_choices: bool = False, z_init=None, noises=None):
        """Autoregressive multi-view generation with STOCHASTIC CONDITIONING.

        views  : (B, k, S, S, 3) known source images in [-1, 1];  poses: dict R (B, k, 3, 3), t (B, k, 3) of those views
        K      : (B, 3, 3) intrinsics;  target_poses: dict R (B, m, 3, 3), t (B, m, 3)
        For each of the m target poses in turn the chain starts from noise and, at EVERY denoising step, conditions on
        one view drawn uniformly from the pool (the k sources plus -- if condition_on_generated -- the targets generated
        so far), exactly as the paper's sampler; one 2B-batch forward per step ([cond ; uncond], guidance weight w) and
        the same posterior update as `sample()`.  The pool lives on the device; a step only copies the chosen view and
        its pose into the engine's static input buffers, so the per-step CUDA graph is shared with `sample()`'s
        non-static path.  z_init (m, B,S,S,3) / noises (m, steps, B,S,S,3) make a run reproducible against the oracle;
        with one source, one target and the same seed the result equals `sample()`.
        Returns (B, m, S, S, 3) [and the (m, steps) pool indices that were drawn]."""
        B, S, e = self.B, self.S, self.eng
        dev = self.dev
        f32 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float32).to(dev)
        pool_x = [v for v in f32(views).unbind(1)]                     # each (B,S,S,3)
        pool_R = [v for v in f32(poses['R']).unbind(1)]
        pool_t = [v for v in f32(poses['t']).unbind(1)]
        tR, tt = f32(target_poses['R']), f32(target_poses['t'])
        m = tR.shape[1]
        Kd = f32(K)
        rng = np.random.RandomState(seed)
        sc = self.sched
        n = B * S * S * 3
        e.inp['K'].copy_(torch.cat([Kd, Kd], 0).reshape(e.inp['K'].shape))
        e.inp['cond_mask'].copy_(torch.cat([torch.ones(B, device=dev), torch.zeros(B, device=dev)]))
        self.lib.xunet_set_static_conditioning(e.h, 0)                  # the conditioning view changes every step
        outs, choices = [], []
        for j in range(m):
            e.inp['R2'].copy_(torch.cat([tR[:, j], tR[:, j]], 0).reshape(e.inp['R2'].shape))
            e.inp['t2'].copy_(torch.cat([tt[:, j], tt[:, j]], 0).reshape(e.inp['t2'].shape))
            if z_init is None:
                g = torch.Generator(device=dev).manual_seed(seed + 7919 * j)
                self.z.copy_(torch.randn(self.z.shape, generator=g, device=dev))
            else:
                self.z.copy_(f32(z_init[j]))
            logsnr = -20.0
            row = []
            for i in range(len(sc) - 1, -1, -1):
                c = int(rng.randint(len(pool_x)))
                row.append(c)
                e.inp['x'].copy_(torch.cat([pool_x[c], pool_x[c]], 0).reshape(e.inp['x'].shape))
                e.inp['R1'].copy_(torch.cat([pool_R[c], pool_R[c]], 0).reshape(e.inp['R1'].shape))
                e.inp['t1'].copy_(torch.cat([pool_t[c], pool_t[c]], 0).reshape(e.inp['t1'].shape))
                e.inp['z'][:B].copy_(self.z)
                e.inp['z'][B:].copy_(self.z)
                e.inp['logsnr'].fill_(float(logsnr))
                self._forward_dynamic()
                sigma = 0.0 if i == 0 else float(np.exp(0.5 * sc.posterior_log_variance_clipped[i]))
                st = torch.cuda.current_stream(dev).cuda_stream
                nz = f32(noises[j][len(sc) - 1 - i]).contiguous() if noises is not None else None
                _lib.check(self.lib.xunet_sampler_update(e.eps.data_ptr(), self.z.data_ptr(), nz.data_ptr() if nz is not None else None,
                                                         self.z.data_ptr(), n, self.w,
                                                         float(sc.sqrt_recip_alphas_cumprod[i]),
                                                         float(sc.sqrt_recipm1_alphas_cumprod[i]),
                                                         float(sc.posterior_mean_coef1[i]), float(sc.posterior_mean_coef2[i]),
                                                         sigma, ((seed + 7919 * j) * 1000003 + i) & 0xFFFFFFFFFFFFFFFF, st),
                           'sampler_update')
                logsnr = logsnr_schedule_cosine(sc.timesteps[i] / 1000.0)
            out = self.z.clone()
            outs.append(out)
            choices.append(row)
            if condition_on_generated:
                pool_x.append(out); pool_R.append(tR[:, j]); pool_t.append(tt[:, j])
        res = torch.stack(outs, 1)
        return (res, np.asarray(choices)) if return_choices else res

    def _forward_dynamic(self):
        """Full forward (rays, posenc, pose convs recomputed): graph-captured once, replayed per step."""
        if not self.use_graph:
            self.eng.forward(self.flat, train=False)
            return
        if getattr(self, 'graph_dyn', None) is None:
            torch.cuda.synchronize(self.dev)
            st = torch.cuda.Stream(device=self.dev)
            with torch.cuda.stream(st):
                self.eng.forward(self.flat, train=False)
                st.synchronize()
                self.graph_dyn = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph_dyn, stream=st):
                    self.eng.forward(self.flat, train=False)
            torch.cuda.synchronize(self.dev)
        self.graph_dyn.replay()


def save_view(path: str, img) -> None:
    """Writes an image in [-1,1] (HWC, RGB) as PNG: the headless replacement of cv2.imshow(z/2+0.5) (sampling.py:153)."""
    import cv2
    a = np.clip(np.asarray(img, dtype=np.float32) / 2.0 + 0.5, 0.0, 1.0)
    cv2.imwrite(path, (a[:, :, ::-1] * 255.0 + 0.5).astype(np.uint8))
