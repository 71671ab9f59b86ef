"""Cost of a sampled view with each sampler: views/s and ms per step of `ddpm` at 256 steps, `ddim` at 50 and `dpmpp_2m` at 25
(log-SNR spacing, so fewer forwards than requested; the forwards actually run are printed), classifier-free guidance w = 3,
CUDA-graph replay.  Per (model, side, views in flight) the three samplers share one engine and are timed alternately, the
order flipped every round (CUDA events around one full `sample()` each); the median over --rounds is printed.  The card
name and power limit are printed first.

    python tools/sampler_cost.py [--rounds 3] [--skip-full]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from oracle import xunet_ref as R
from tools.ema_step_cost import card

METHODS = (('ddpm', 256), ('ddim', 50), ('dpmpp_2m', 25))


def run(label, model, S, views, rounds):
    params = P.create_train_state(0, 1, 1e-4, 1, S, model=model, init_on_device=label == 'full').params
    for B in views:
        batch = {k: v.numpy().astype(np.float32) for k, v in R.synthetic_batch(B, S, seed=1234)[0].items()}
        samplers = {m: P.Sampler(model, params, B, S, steps=n, w=3.0, method=m) for m, n in METHODS}
        for s in samplers.values():
            s.capture(batch)
        torch.cuda.synchronize()
        times = {m: [] for m in samplers}
        keys = list(samplers)
        for r in range(rounds):
            for m in (keys if r % 2 == 0 else keys[::-1]):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                samplers[m].sample(batch, seed=r)
                e1.record()
                e1.synchronize()
                times[m].append(e0.elapsed_time(e1) * 1e-3)
        for (m, n), s in zip(METHODS, samplers.values()):
            t = float(np.median(times[m]))
            f = len(s.sched)
            print(f'{label} {S}x{S} views={B} {m:9s} steps={n:3d} forwards={f:3d}: {B / t:7.3f} views/s, '
                  f'{t / f * 1e3:6.2f} ms/step, {t:7.3f} s/run (min {min(times[m]):.3f}, max {max(times[m]):.3f})', flush=True)
        del samplers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('sampler_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    run('small', P.XUNet(dtype='bf16'), 64, (1, 8), a.rounds)
    if not a.skip_full:
        run('full', P.XUNet.from_config(P.XUNetConfig(**{**P.FULL_3DIM.__dict__, 'dtype': 'bf16'})), 128, (1, 4), a.rounds)


if __name__ == '__main__':
    main()
