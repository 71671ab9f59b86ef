"""Cost of the mean-squared epsilon loss in the fused training step: TrainStep with loss='frobenius' (the default) and with
loss='mse' on the same model and buffers, alternated in one process over several rounds (CUDA events over >= 20 graph
replays after warm-up), for the small 64² model at B = 8 and the full 128² model at B = 4.  The card name and power limit
are printed first.

    python tools/loss_step_cost.py [--steps 20] [--rounds 5] [--skip-full]
"""
import argparse
import os
import sys
from dataclasses import replace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from bench import make_host_batches
from tools.ema_step_cost import card, time_alternating


def train_step(label, cfg, S, B, reps, rounds, init_on_device):
    """One model and one set of buffers; a Frobenius and an MSE TrainStep view of them (they train the same weights: the
    numbers they compute are irrelevant here, only the time is)."""
    model = P.XUNet.from_config(cfg)
    st = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=init_on_device)
    views = {'frobenius': st, 'mse': replace(st, loss='mse', opt_state=replace(st.opt_state))}
    steps = {k: P.TrainStep(s) for k, s in views.items()}
    (batch, noise), = make_host_batches(1, B, S, 1234)
    cond = np.ones(B, np.float32)
    fns = {k: (lambda s=s: s(batch, noise, cond_mask=cond)) for k, s in steps.items()}
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    a = t['frobenius'][0]
    print(f'{label}: {st.params.flat.numel()} parameters, B={B}, {S}x{S}, {cfg.dtype}, {reps} steps x {rounds} rounds per arm')
    for k, (med, lo, hi) in t.items():
        d = '' if k == 'frobenius' else f'   {med - a:+.3f} ms = {100 * (med - a) / a:+.2f} %'
        print(f'  {k:9s} {med:9.3f} ms/step  (min {lo:.3f}, max {hi:.3f}){d}')
    del steps, views, st, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('loss_step_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    train_step('small', P.SMALL, 64, 8, max(a.steps, 20), max(a.rounds, 5), init_on_device=False)
    if not a.skip_full:
        train_step('full', P.FULL_3DIM, 128, 4, max(a.steps, 20), max(a.rounds, 5), init_on_device=True)


if __name__ == '__main__':
    main()
