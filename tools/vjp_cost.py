"""Cost of the vector-Jacobian product: forward + Engine.backward_vjp (parameter gradient only, and with dx and dz) against
forward + Engine.backward(loss='mse') on the same engine and buffers, eager calls alternated in one process (CUDA events,
median over rounds), for the small 64² model at B = 8 and the full 128² model at B = 4; then the input-gradient kernel alone
(conv_cin3_dgrad_unpack_kernel, torch.profiler device time per launch, in a child process with XUNET_NO_PDL=1 so a kernel's
span does not include the time it waits behind its predecessor).  The card name and power limit are printed first.

    python tools/vjp_cost.py [--reps 10] [--rounds 5] [--skip-full]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from bench import make_host_batches
from tools.ema_step_cost import card, time_alternating

KERNEL = 'conv_cin3_dgrad_unpack_kernel'


def setup(cfg, S, B):
    model = P.XUNet.from_config(cfg)
    init_on_device = cfg.ch >= 256
    flat = model.init({'params': 0}, {'x': np.zeros((B, S, S, 3))}, zero_init=False, on_device=init_on_device)['params'].flat
    eng = model.engine(B, S, True)
    (batch, noise), = make_host_batches(1, B, S, 1234)
    eng.load_inputs(batch, cond_mask=np.ones(B, np.float32), noise=noise)
    d_eps = torch.randn(B, S, S, 3, device=eng.device, generator=torch.Generator(eng.device).manual_seed(1))
    return model, flat, eng, d_eps


def arms(flat, eng, d_eps):
    def fwd():
        eng.forward(flat, train=True)
    return {
        'fwd+bwd(mse)': lambda: (fwd(), eng.backward(flat, loss='mse')),
        'fwd+vjp': lambda: (fwd(), eng.backward_vjp(flat, d_eps)),
        'fwd+vjp+dx+dz': lambda: (fwd(), eng.backward_vjp(flat, d_eps, dx=True, dz=True)),
    }


def end_to_end(label, cfg, S, B, reps, rounds):
    model, flat, eng, d_eps = setup(cfg, S, B)
    fns = arms(flat, eng, d_eps)
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    a = t['fwd+bwd(mse)'][0]
    print(f'{label}: {flat.numel()} parameters, B={B}, {S}x{S}, {cfg.dtype}, {reps} calls x {rounds} rounds per arm')
    for k, (med, lo, hi) in t.items():
        d = '' if k == 'fwd+bwd(mse)' else f'   {med - a:+.3f} ms = {100 * (med - a) / a:+.2f} %'
        print(f'  {k:14s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f}){d}')
    del eng, model
    torch.cuda.empty_cache()


def kernel_alone(label, cfg, S, B, reps):
    model, flat, eng, d_eps = setup(cfg, S, B)
    f = arms(flat, eng, d_eps)['fwd+vjp+dx+dz']
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            f()
        torch.cuda.synchronize()
    times = [(e.key, getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0)), e.count) for e in prof.key_averages()
             if KERNEL in e.key]
    if not times:
        raise SystemExit(f'{KERNEL} not found in the profile')
    tot = sum(t for _, t, _ in times)
    n = sum(c for _, _, c in times)
    # bytes it must move: the (2B,S,S,ch) output gradient of the input conv read once, dx and dz written once
    act = 4 if cfg.dtype == 'fp32' else 2
    nbytes = 2 * B * S * S * cfg.ch * act + 2 * B * S * S * 3 * 4
    us = tot / n
    print(f'{label}: {KERNEL} {us:.2f} us per launch over {n} launches; {nbytes / 1e6:.2f} MB -> {nbytes / us / 1e3:.0f} GB/s')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--skip-full', action='store_true')
    ap.add_argument('--kernel-only', action='store_true', help='(child process) profile the input-gradient kernel alone')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('vjp_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    shapes = [('small', P.SMALL, 64, 8)] + ([] if a.skip_full else [('full', P.FULL_3DIM, 128, 4)])
    if a.kernel_only:
        for label, cfg, S, B in shapes:
            kernel_alone(label, cfg, S, B, a.reps)
        return
    print(card())
    for label, cfg, S, B in shapes:
        end_to_end(label, cfg, S, B, a.reps, a.rounds)
    cmd = [sys.executable, os.path.abspath(__file__), '--kernel-only', '--reps', str(a.reps)] + (['--skip-full'] if a.skip_full else [])
    sys.stdout.flush()
    subprocess.run(cmd, check=True, env=dict(os.environ, XUNET_NO_PDL='1'))


if __name__ == '__main__':
    main()
