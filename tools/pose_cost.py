"""Cost of one pose-estimation iteration (pose.PoseEstimator): the iteration's CUDA graph (draw, forward, loss, camera VJP,
tangent, Adam, retraction, count) against a graph of the forward + Engine.backward_vjp_inputs(cameras=True) alone on the same
engine, slots and batch B = H P, replays alternated in one process (CUDA events, median over rounds).  Small 64^2 model with
H P = 8 (H = 4, P = 2) and the full 3DiM 128^2 model with H P = 4 (H = 2, P = 2), bf16, freshly initialised weights.  The card
name and power limit are printed first.

    python tools/pose_cost.py [--reps 20] [--rounds 7] [--skip-full]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import pose as PO
from tools.ema_step_cost import card, time_alternating


def _capture(fn):
    side = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        fn()
    return g


def measure(label, cfg, S, H, Pd, reps, rounds):
    model = P.XUNet.from_config(cfg)
    params = model.init({'params': 0}, {'x': np.zeros((1, S, S, 3))}, zero_init=False, on_device=cfg.ch >= 256)['params']
    est = PO.PoseEstimator(model, params, S, hypotheses=H, draws=Pd)
    rng = np.random.RandomState(0)
    c = np.array([0.3, -0.8, 0.9])
    c = 1.3 * c / np.linalg.norm(c)
    f = 131.25 * S / 128
    K = np.array([[f, 0, S / 2], [0, f, S / 2], [0, 0, 1.0]])
    R1 = PO.sphere_init(np.eye(3), c, 1)[0][0]
    est.estimate(rng.uniform(-1, 1, (S, S, 3)), R1, c, K, rng.uniform(-1, 1, (S, S, 3)), iters=2)   # slots, views, warm-up
    loss = torch.zeros(1, H, device=est.dev)
    it = _capture(lambda: est._iteration(0, loss))
    eng = est.eng
    base = _capture(lambda: (eng.forward(est.flat, train=False, inputs=(est.slots, 0)),
                             eng.backward_vjp_inputs(est.flat, est.d_eps, cameras=True, inputs=(est.slots, 0))))
    fns = {'fwd+vjp_inputs(cameras)': base.replay, 'pose iteration': it.replay}
    for fn in fns.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    a = t['fwd+vjp_inputs(cameras)'][0]
    print(f'{label}: {est.flat.numel()} parameters, H={H} x P={Pd} = B {H * Pd}, {S}x{S}, {cfg.dtype}, graph replays, '
          f'{reps} x {rounds} rounds per arm')
    for k, (med, lo, hi) in t.items():
        d = '' if k == 'fwd+vjp_inputs(cameras)' else f'   {med - a:+.4f} ms = {100 * (med - a) / a:+.2f} %'
        print(f'  {k:24s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f}){d}')
    del it, base, est, eng, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('pose_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    measure('small 64^2', P.SMALL, 64, 4, 2, a.reps, a.rounds)
    if not a.skip_full:
        measure('full 3DiM 128^2', P.FULL_3DIM, 128, 2, 2, a.reps, a.rounds)


if __name__ == '__main__':
    main()
