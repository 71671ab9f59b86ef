"""Cost of gradient accumulation in the fused training step: ms per update and images/s of TrainStep at grad_accum_steps
k = 1, 2, 4 on one model and one set of buffers, the values of k alternated over several rounds (CUDA events over graph
replays after warm-up), next to k x the k = 1 step minus (k - 1) Adam passes (the cost if the only saving were the
per-update fixed work).

    python tools/accum_step_cost.py [--steps 10] [--rounds 5] [--skip-full]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from bench import make_host_batches
from tools.ema_step_cost import card, time_alternating

KS = (1, 2, 4)


def adam_ms(st, reps):
    """One Adam pass over the state's flat buffers (what a k-step update runs once instead of k times)."""
    g = torch.zeros_like(st.params.flat)
    s = st.apply_gradients(grads=g, copy=True)        # a copy: the timed passes must not move the trained weights
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        s.apply_gradients(grads=g)
    b.record()
    torch.cuda.synchronize()
    del s, g
    return a.elapsed_time(b) / reps


def train_step(label, cfg, S, B, reps, rounds, init_on_device):
    model = P.XUNet.from_config(cfg)
    st = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=init_on_device)
    steps = {k: P.TrainStep(st, grad_accum_steps=k) for k in KS}
    (batch, noise), = make_host_batches(1, max(KS) * B, S, 1234)
    fns = {}
    for k, s in steps.items():
        bk = {key: v[:k * B] for key, v in batch.items()}
        fns[k] = (lambda s=s, bk=bk, nk=noise[:k * B], ck=np.ones(k * B, np.float32): s(bk, nk, cond_mask=ck))
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    t_adam = adam_ms(st, reps)
    n = st.params.flat.numel()
    one = t[1][0]
    print(f'{label}: {n} parameters, B={B} per micro-batch, {S}x{S}, {cfg.dtype}, {reps} updates x {rounds} rounds per arm; '
          f'Adam pass alone {t_adam:.3f} ms')
    for k, (med, lo, hi) in t.items():
        naive = k * one - (k - 1) * t_adam
        print(f'  k={k}  {med:9.3f} ms/update  (min {lo:.3f}, max {hi:.3f})  {k * B / med * 1e3:8.1f} images/s  '
              f'k x step(k=1) - (k-1) x Adam = {naive:9.3f} ms')
    del steps, st, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('accum_step_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    train_step('small', P.SMALL, 64, 8, max(a.steps, 20), a.rounds, init_on_device=False)
    if not a.skip_full:
        train_step('full', P.FULL_3DIM, 128, 4, a.steps, a.rounds, init_on_device=True)


if __name__ == '__main__':
    main()
