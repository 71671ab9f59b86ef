"""Device-side forward diffusion (SURVEY 8(f) row 2): the per-item noise / timestep / z / logsnr / cond_mask work that the
reference does on the host inside SceneInstanceDataset.__getitem__ (dataset/data_loader.py:70-74, 88-110) and train.py:64.

    fd = ForwardDiffusion(engine)                 # uploads the cosine-beta tables once
    fd.sample(x0_target, seed)                    # fills engine.inp['z'], ['noise'], ['logsnr'], ['cond_mask'] on the GPU
Only the clean source / target images and the poses then cross PCIe (no z, no noise).

With min_snr_gamma set, sample() also fills engine.inp['loss_weight'] (= fd.loss_weight) with the min-SNR-gamma weights of
the drawn timesteps (Hang et al. 2023), for a state built with loss='mse'.

With prediction='v', sample() writes the v target v = sqrt(abar_t) noise - sqrt(1 - abar_t) x0 (Salimans & Ho 2022) into
engine.inp['noise'] in place of the noise, in the same kernel (xunet_forward_diffusion_v): the buffer the loss regresses the
network output onto.  v_target() restates that kernel in numpy, bit for bit."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from .sampling import check_prediction, cosine_beta_schedule


def min_snr_weights(gamma: float, timesteps: int = 1000, prediction: str = 'eps') -> np.ndarray:
    """Per-timestep min-SNR-gamma loss weights (Hang et al. 2023) for t = 0..timesteps-1 (float64): min(SNR_t, gamma) / SNR_t
    for an eps-prediction model, min(SNR_t, gamma) / (SNR_t + 1) for a v-prediction one, with SNR_t = alpha_bar_t /
    (1 - alpha_bar_t) from the cosine-beta table that noises z (data_loader.py:15-25,70-74) -- not from the batch's logsnr,
    which follows the logsnr-cosine schedule and disagrees with it near both ends."""
    check_prediction(prediction)
    gamma = float(gamma)
    if not (gamma > 0.0 and np.isfinite(gamma)):
        raise ValueError(f'min_snr_gamma must be a finite number > 0, got {gamma}')
    ac = np.cumprod(1. - cosine_beta_schedule(timesteps), axis=0)
    snr = ac / (1. - ac)
    return np.minimum(snr, gamma) / (snr if prediction == 'eps' else snr + 1.)


def diffusion_tables(timesteps: int = 1000):
    """The fp32 tables (sqrt(alpha_bar_t), sqrt(1 - alpha_bar_t)) of the cosine-beta schedule, t = 0..timesteps-1, that the
    forward-diffusion kernels read: z = sqrt_ac[t] x0 + sqrt_1mac[t] noise (data_loader.py:73-74)."""
    ac = np.cumprod(1. - cosine_beta_schedule(timesteps), axis=0)
    return np.sqrt(ac).astype(np.float32), np.sqrt(1. - ac).astype(np.float32)


def v_target(x0, noise, t) -> np.ndarray:
    """The v-prediction target v = alpha_t noise - sigma_t x0 (Salimans & Ho 2022) with alpha_t = sqrt_ac[t] and
    sigma_t = sqrt_1mac[t] (diffusion_tables), in fp32 with each product and the difference rounded once: bit for bit what
    xunet_forward_diffusion_v and xunet_srn_batch_v store.  x0, noise: (B, ...); t: (B,) integer timesteps."""
    sa, sb = diffusion_tables()
    t = np.asarray(t, dtype=np.int64)
    x0, noise = np.asarray(x0, dtype=np.float32), np.asarray(noise, dtype=np.float32)
    shape = (len(t),) + (1,) * (x0.ndim - 1)
    return sa[t].reshape(shape) * noise - sb[t].reshape(shape) * x0


class ForwardDiffusion:
    def __init__(self, engine, p_uncond: float = 0.1, min_snr_gamma: Optional[float] = None, prediction: str = 'eps'):
        """prediction: the target sample() writes to engine.inp['noise']: 'eps' (the noise) or 'v' (the v target, for a
        state built with prediction='v'); min_snr_gamma weights follow it (min_snr_weights)."""
        self.eng, self.lib, self.p_uncond = engine, _lib.load(), float(p_uncond)
        self.prediction = check_prediction(prediction)
        sqrt_ac, sqrt_1mac = diffusion_tables()
        dev = engine.device
        self.sqrt_ac = torch.as_tensor(sqrt_ac).to(dev)               # data_loader.py:73
        self.sqrt_1mac = torch.as_tensor(sqrt_1mac).to(dev)           # data_loader.py:74
        self.t = torch.zeros(engine.B, dtype=torch.int32, device=dev)
        self.x0 = torch.zeros_like(engine.inp['z'])
        # v mode: explicit noise is staged here, since engine.inp['noise'] receives v
        self.noise = torch.zeros_like(engine.inp['z']) if prediction == 'v' else engine.inp['noise']
        # per-timestep min-SNR-gamma weights, gathered by the device t of each sample (None: no weighting)
        self.snr_weight = None if min_snr_gamma is None else \
            torch.as_tensor(min_snr_weights(min_snr_gamma, prediction=prediction), dtype=torch.float32).to(dev)
        self.loss_weight = None if min_snr_gamma is None else engine.inp['loss_weight']

    def sample(self, x0, seed: int, *, t=None, noise=None) -> None:
        """x0: clean target images (B,S,S,3), host or device.  t / noise: optional fixed timesteps / noise (parity tests)."""
        e = self.eng
        src = x0 if isinstance(x0, torch.Tensor) else torch.as_tensor(np.asarray(x0), dtype=torch.float32)
        self.x0.copy_(src.reshape(self.x0.shape).to(torch.float32), non_blocking=True)
        t_ptr = n_ptr = None
        if t is not None:
            self.t.copy_(torch.as_tensor(np.asarray(t), dtype=torch.int32))
            t_ptr = self.t.data_ptr()
        if noise is not None:
            self.noise.copy_(torch.as_tensor(np.asarray(noise), dtype=torch.float32).reshape(self.noise.shape))
            n_ptr = self.noise.data_ptr()
        per = e.S * e.S * 3
        st = torch.cuda.current_stream(e.device).cuda_stream
        head = (self.x0.data_ptr(), n_ptr, t_ptr, int(seed) & 0xFFFFFFFFFFFFFFFF, self.sqrt_ac.data_ptr(),
                self.sqrt_1mac.data_ptr(), self.p_uncond, e.inp['z'].data_ptr())
        tail = (e.inp['logsnr'].data_ptr(), self.t.data_ptr() if t is None else None, e.inp['cond_mask'].data_ptr(), e.B, per,
                st)
        if self.prediction == 'v':
            _lib.check(self.lib.xunet_forward_diffusion_v(*head, None, e.inp['noise'].data_ptr(), *tail),
                       'xunet_forward_diffusion_v')
        else:
            _lib.check(self.lib.xunet_forward_diffusion(*head, e.inp['noise'].data_ptr(), *tail), 'xunet_forward_diffusion')
        if self.snr_weight is not None:
            self.loss_weight.copy_(self.snr_weight[self.t.long()])
