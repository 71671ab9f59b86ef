"""Image-quality metrics of generated views against held-out ground truth: per-image MSE, PSNR and SSIM, computed on the GPU by
xunet_image_metrics (include/xunet_b200.h states the exact definitions; SSIM is the Gaussian-window SSIM of Wang et al. 2004
that 3DiM and pixelNeRF report on SRN).

    m = image_metrics(views, target)      # (B,S,S,3) in [-1, 1], e.g. straight from Sampler.sample
    m['psnr'].mean().item(), m['ssim'].mean().item()
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from . import _lib

MAX_SIDE = 256   # XUNET_METRICS_MAX_SIDE


def _as_device_f32(a, name: str, device) -> torch.Tensor:
    t = a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a))
    if t.ndim != 4 or t.shape[1] != t.shape[2] or t.shape[3] != 3:
        raise ValueError(f'{name}: expected shape (B, S, S, 3), got {tuple(t.shape)}')
    return t.to(device=device, dtype=torch.float32).contiguous()


def image_metrics(pred, target) -> Dict[str, torch.Tensor]:
    """Per-image {'mse', 'psnr', 'ssim'}, each a (B,) float32 tensor on the current CUDA device.

    pred, target: (B,S,S,3) images in [-1, 1] (values are clamped to it), torch tensors on any device or numpy arrays; they are
    made contiguous fp32 on the current CUDA device.  The kernel is launched on the current stream and nothing synchronises, so
    the call can be captured in a CUDA graph.  PSNR uses data range 1 after mapping [-1, 1] to [0, 1] and is +inf for identical
    images.  Raises ValueError for mismatched or non-(B,S,S,3) shapes and for S outside [11, MAX_SIDE]."""
    dev = torch.device('cuda', torch.cuda.current_device())
    p = _as_device_f32(pred, 'pred', dev)
    t = _as_device_f32(target, 'target', dev)
    if p.shape != t.shape:
        raise ValueError(f'pred {tuple(p.shape)} and target {tuple(t.shape)} differ in shape')
    B, S = p.shape[0], p.shape[1]
    if B < 1 or not 11 <= S <= MAX_SIDE:
        raise ValueError(f'need B >= 1 and 11 <= S <= {MAX_SIDE}, got B={B}, S={S}')
    out = torch.empty(3, B, dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    _lib.check(_lib.load().xunet_image_metrics(p.data_ptr(), t.data_ptr(), B, S, out[0].data_ptr(), out[1].data_ptr(),
                                               out[2].data_ptr(), st), 'xunet_image_metrics')
    return {'mse': out[0], 'psnr': out[1], 'ssim': out[2]}
