"""Cost of gradient clipping by global norm and learning-rate warm-up in the fused training step: the norm kernel alone and
the clip / warm-up Adam launch against the plain Adam launch, through the C-ABI at the full-model parameter count (with the
achieved HBM bandwidth over the bytes each must move), and TrainStep with and without the features in one process,
alternated over several rounds (CUDA events over >= 20 graph replays after warm-up).

    python tools/clip_step_cost.py [--steps 20] [--rounds 5] [--skip-full]
"""
import argparse
import os
import sys
from dataclasses import replace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200.train import ClipState
from bench import make_host_batches
from tools.ema_step_cost import N_FULL, BYTES_ADAM, card, time_alternating

BYTES_NORM = 4                              # per parameter: g read once more


def kernels_alone(reps, rounds):
    lib = _lib.load()
    n = N_FULL
    p, g, m, v = (torch.randn(n, device='cuda') * 1e-2 for _ in range(4))
    scratch = torch.zeros(_lib.GRAD_NORM_SCRATCH, dtype=torch.float64, device='cuda')
    norm = torch.zeros(1, device='cuda')
    skipped = torch.zeros(1, dtype=torch.int64, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    ptrs = (p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr())
    fns = {
        'norm': lambda: _lib.check(lib.xunet_grad_global_norm(g.data_ptr(), n, 1.0, scratch.data_ptr(), norm.data_ptr(), st)),
        'adam': lambda: _lib.check(lib.xunet_adam_step(*ptrs, n, 1, None, 1e-4, 0.9, 0.999, 1e-8, 1.0, st)),
        # the norm of these gradients is ~100: max_norm 1 clips every element
        'clip-adam': lambda: _lib.check(lib.xunet_adam_clip_step(*ptrs, None, n, 5, None, 1e-4, 0.9, 0.999, 1e-8, 1.0, 0.0,
                                                                 norm.data_ptr(), 1.0, 10, skipped.data_ptr(), st)),
    }
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    assert float(norm) > 1.0 and int(skipped) == 0
    t = time_alternating(fns, reps, rounds)
    del p, g, m, v
    torch.cuda.empty_cache()
    print(f'Kernels alone, n = {n} parameters:')
    for k, b in (('norm', BYTES_NORM), ('adam', BYTES_ADAM), ('clip-adam', BYTES_ADAM)):
        med, lo, hi = t[k]
        print(f'  {k:9s} {med:8.3f} ms  (min {lo:.3f}, max {hi:.3f})  {b * n / med / 1e6:7.0f} GB/s over {b} B/param')
    extra = t['norm'][0] + t['clip-adam'][0] - t['adam'][0]
    print(f'  clipping adds {extra:.3f} ms per update (norm + clip-adam - adam; the extra read of g is {BYTES_NORM * n / 1e9:.3f} GB, '
          f'>= {BYTES_NORM * n / 3.35e12 * 1e3:.2f} ms at the 3.35 TB/s data-sheet rate)')


def train_step(label, cfg, S, B, reps, rounds, init_on_device):
    """One model and one set of buffers; TrainStep views of them with plain Adam, with warm-up only, and with clipping and
    warm-up.  They all train the same weights (the numbers they compute are irrelevant here; only the time is)."""
    model = P.XUNet.from_config(cfg)
    st_plain = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=init_on_device)
    clip = ClipState.zeros(st_plain.params.flat.device)
    views = {
        'plain': st_plain,
        'warm-up': replace(st_plain, tx=replace(st_plain.tx, warmup_steps=5000), clip=clip, opt_state=replace(st_plain.opt_state)),
        'clip+warm-up': replace(st_plain, tx=replace(st_plain.tx, max_grad_norm=1.0, warmup_steps=5000), clip=clip,
                                opt_state=replace(st_plain.opt_state)),
    }
    steps = {k: P.TrainStep(s) for k, s in views.items()}
    (batch, noise), = make_host_batches(1, B, S, 1234)
    cond = np.ones(B, np.float32)
    fns = {k: (lambda s=s: s(batch, noise, cond_mask=cond)) for k, s in steps.items()}
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    n = st_plain.params.flat.numel()
    a = t['plain'][0]
    print(f'{label}: {n} parameters, B={B}, {S}x{S}, {cfg.dtype}, {reps} steps x {rounds} rounds per arm')
    for k, (med, lo, hi) in t.items():
        d = '' if k == 'plain' else f'   {med - a:+.3f} ms = {100 * (med - a) / a:+.2f} %'
        print(f'  {k:13s} {med:9.3f} ms/step  (min {lo:.3f}, max {hi:.3f}){d}')
    del steps, views, st_plain, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('clip_step_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    kernels_alone(max(a.steps, 20), max(a.rounds, 5))
    train_step('small', P.SMALL, 64, 8, a.steps, max(a.rounds, 5), init_on_device=False)
    if not a.skip_full:
        train_step('full', P.FULL_3DIM, 128, 4, a.steps, max(a.rounds, 5), init_on_device=True)


if __name__ == '__main__':
    main()
