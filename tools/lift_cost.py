"""Cost of one lifting iteration (lift.FieldLifter): the iteration's CUDA graph (draw, render of P + 1 views, noise, the guided
2P forward, image gradient, render backward, Adam on the grid, count) against a graph of the 2P forward alone on the same
engine and slots, replays alternated in one process (CUDA events, median over rounds).  Small 64^2 model with P = 4 and G = 64,
and the full 3DiM 128^2 model with P = 2 and G = 128, bf16, freshly initialised weights.  The card name and power limit are
printed first.

    python tools/lift_cost.py [--reps 20] [--rounds 7] [--skip-full]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import lift as LI
from novel_view_synthesis_3d_b200.synthetic import _look_at
from tools.ema_step_cost import card, time_alternating


def _capture(fn):
    side = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        fn()
    return g


def measure(label, cfg, S, Pd, G, reps, rounds):
    model = P.XUNet.from_config(cfg)
    params = model.init({'params': 0}, {'x': np.zeros((1, S, S, 3))}, zero_init=False, on_device=cfg.ch >= 256)['params']
    lf = LI.FieldLifter(model, params, S, draws=Pd, grid=G)
    rng = np.random.RandomState(0)
    c = np.array([0.3, -0.8, 0.9])
    c = 1.3 * c / np.linalg.norm(c)
    f = 131.25 * S / 128
    K = np.array([[f, 0, S / 2], [0, f, S / 2], [0, 0, 1.0]])
    lf.lift(rng.uniform(-1, 1, (S, S, 3)), _look_at(c), c, K, iters=2)       # slots, cameras, warm-up
    sds, loss = torch.zeros(1, device=lf.dev), torch.zeros(1, device=lf.dev)
    it = _capture(lambda: lf._iteration(lf._a, sds, loss))
    base = _capture(lambda: lf.eng.forward(lf.flat, train=False, inputs=(lf.slots, 0)))
    fns = {'2P forward': base.replay, 'lift iteration': it.replay}
    for fn in fns.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    a = t['2P forward'][0]
    print(f'{label}: {lf.flat.numel()} parameters, P={Pd} (batch {2 * Pd}), {S}x{S}, G={G}, {cfg.dtype}, graph replays, '
          f'{reps} x {rounds} rounds per arm')
    for k, (med, lo, hi) in t.items():
        d = '' if k == '2P forward' else f'   {med - a:+.4f} ms = {100 * (med - a) / a:+.2f} %'
        print(f'  {k:16s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f}){d}')
    del it, base, lf, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('lift_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    measure('small 64^2', P.SMALL, 64, 4, 64, a.reps, a.rounds)
    if not a.skip_full:
        measure('full 3DiM 128^2', P.FULL_3DIM, 128, 2, 128, a.reps, a.rounds)


if __name__ == '__main__':
    main()
