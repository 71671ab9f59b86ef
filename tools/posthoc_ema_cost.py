"""Cost of the post-hoc EMA (two power-function averages) fused into the Adam kernel, against plain Adam and the fixed-decay
EMA, all in one process and alternated (CUDA events over >= 20 launches or graph replays after warm-up):

  - the Adam launch alone through the C-ABI at the full-model parameter count, with the HBM bandwidth it achieves over
    the bytes it must move (28 / 36 / 44 per parameter);
  - the captured TrainStep, small 64x64 B = 8 and full 128x128 B = 4, without an EMA, with ema_decay and with posthoc_ema.
    The three steps share one set of parameters and Adam moments: only the time is compared.

    python tools/posthoc_ema_cost.py [--steps 20] [--rounds 5] [--skip-full]
"""
import argparse
import os
import sys
from dataclasses import replace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200.posthoc import sigma_rel_to_gamma
from bench import make_host_batches
from ema_step_cost import card, time_alternating

N_FULL = 438831363                          # FULL_3DIM at 128x128
BYTES = {'adam': 28, 'adam+ema': 36, 'adam+posthoc': 44}    # per parameter: p, m, v read + written, g read; +8 per average


def adam_alone(reps, rounds):
    lib = _lib.load()
    n = N_FULL
    p, g, m, v, e, eb = (torch.randn(n, device='cuda') * 1e-2 for _ in range(6))
    st = torch.cuda.current_stream().cuda_stream
    ga, gb = sigma_rel_to_gamma(0.05), sigma_rel_to_gamma(0.10)
    fns = {
        'adam': lambda: _lib.check(lib.xunet_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, 1000, None,
                                                       1e-4, 0.9, 0.999, 1e-8, 1.0, st)),
        'adam+ema': lambda: _lib.check(lib.xunet_adam_ema_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(),
                                                               e.data_ptr(), n, 1000, None, 1e-4, 0.9, 0.999, 1e-8, 1.0,
                                                               0.9999, st)),
        'adam+posthoc': lambda: _lib.check(lib.xunet_adam_posthoc_step(p.data_ptr(), g.data_ptr(), m.data_ptr(),
                                                                       v.data_ptr(), e.data_ptr(), eb.data_ptr(), n, 1000,
                                                                       None, 1e-4, 0.9, 0.999, 1e-8, 1.0, ga, gb, None,
                                                                       0.0, 0, None, st)),
    }
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    del p, g, m, v, e, eb
    torch.cuda.empty_cache()
    print(f'Adam launch alone, n = {n} parameters:')
    for k, (med, lo, hi) in t.items():
        print(f'  {k:13s} {med:8.3f} ms  (min {lo:.3f}, max {hi:.3f})  {BYTES[k] * n / med / 1e6:7.0f} GB/s over '
              f'{BYTES[k]} B/param')
    ta = t['adam'][0]
    print(f'  vs plain Adam: EMA {t["adam+ema"][0] - ta:+.3f} ms, post-hoc {t["adam+posthoc"][0] - ta:+.3f} ms')


def train_step(label, cfg, S, B, reps, rounds, init_on_device):
    model = P.XUNet.from_config(cfg)
    st_ph = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=init_on_device, posthoc_ema=(0.05, 0.10))
    ema = model.tree_from_flat(st_ph.params.flat.clone(), S, B)
    st_plain = replace(st_ph, posthoc=None, opt_state=replace(st_ph.opt_state))
    st_ema = replace(st_ph, posthoc=None, ema_params=ema, ema_decay=0.9999, opt_state=replace(st_ph.opt_state))
    steps = {'no EMA': P.TrainStep(st_plain), 'ema_decay': P.TrainStep(st_ema), 'posthoc_ema': P.TrainStep(st_ph)}
    (batch, noise), = make_host_batches(1, B, S, 1234)
    cond = np.ones(B, np.float32)
    fns = {k: (lambda s=s: s(batch, noise, cond_mask=cond)) for k, s in steps.items()}
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    n = st_ph.params.flat.numel()
    a = t['no EMA'][0]
    print(f'{label}: {n} parameters, B={B}, {S}x{S}, {cfg.dtype}, {reps} steps x {rounds} rounds per arm')
    for k, (med, lo, hi) in t.items():
        print(f'  {k:11s} {med:9.3f} ms/step  (min {lo:.3f}, max {hi:.3f})  {100 * (med - a) / a:+.2f} %')
    del steps, st_plain, st_ema, st_ph, ema, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('posthoc_ema_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    adam_alone(max(a.steps, 20), a.rounds)
    train_step('small', P.SMALL, 64, 8, a.steps, a.rounds, init_on_device=False)
    if not a.skip_full:
        train_step('full', P.FULL_3DIM, 128, 4, a.steps, a.rounds, init_on_device=True)
    print(card())


if __name__ == '__main__':
    main()
