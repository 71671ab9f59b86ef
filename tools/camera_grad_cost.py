"""Cost of the camera gradient: forward + Engine.backward_vjp (parameter gradient) against forward +
Engine.backward_vjp_inputs(cameras=True) (the same plus d_rays, dR, dt, dK) on the same engine, eager calls alternated in one
process (CUDA events, median over rounds), for the small 64² model at B = 8 and the full 128² model at B = 4, bf16; then the new
kernels alone (torch.profiler device time per call, in a child process with XUNET_NO_PDL=1) with the achieved TFLOP/s of the
pose-embedding data gradients they compute (2 x input pixels reached x taps x 144 x emb_ch per level, from the shapes).  The card
name and power limit are printed first.

    python tools/camera_grad_cost.py [--reps 10] [--rounds 5] [--skip-full]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import novel_view_synthesis_3d_b200 as P
from tools.ema_step_cost import card, time_alternating
from tools.vjp_cost import setup

KERNELS = ('pose_dgrad_tc_kernel', 'pose_dgrad_simt_kernel', 'camera_grad_kernel')


def dgrad_flops(cfg, S, B):
    """Multiply-adds x 2 of the pose-embedding data gradients: every output pixel of level l feeds 9 taps x 144 x emb_ch."""
    return sum(2.0 * 2 * B * (S >> l) ** 2 * 9 * 144 * cfg.emb_ch for l in range(len(cfg.ch_mult)))


def arms(flat, eng, d_eps):
    def fwd():
        eng.forward(flat, train=True)
    return {
        'fwd+vjp': lambda: (fwd(), eng.backward_vjp(flat, d_eps)),
        'fwd+vjp+cameras': lambda: (fwd(), eng.backward_vjp_inputs(flat, d_eps, cameras=True)),
    }


def end_to_end(label, cfg, S, B, reps, rounds):
    model, flat, eng, d_eps = setup(cfg, S, B)
    fns = arms(flat, eng, d_eps)
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    a = t['fwd+vjp'][0]
    print(f'{label}: {flat.numel()} parameters, B={B}, {S}x{S}, {cfg.dtype}, {reps} calls x {rounds} rounds per arm')
    for k, (med, lo, hi) in t.items():
        d = '' if k == 'fwd+vjp' else f'   {med - a:+.3f} ms = {100 * (med - a) / a:+.2f} %'
        print(f'  {k:16s} {med:9.3f} ms  (min {lo:.3f}, max {hi:.3f}){d}')
    del eng, model
    torch.cuda.empty_cache()


def kernels_alone(label, cfg, S, B, reps):
    model, flat, eng, d_eps = setup(cfg, S, B)
    f = arms(flat, eng, d_eps)['fwd+vjp+cameras']
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            f()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                per[k] = per.get(k, 0.0) + getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0)) / reps
    if 'pose_dgrad_tc_kernel' not in per:
        raise SystemExit('pose_dgrad_tc_kernel not found in the profile')
    fl = dgrad_flops(cfg, S, B)
    dg = per.get('pose_dgrad_tc_kernel', 0.0) + per.get('pose_dgrad_simt_kernel', 0.0)
    print(f'{label}: ' + ', '.join(f'{k} {v:.1f} us' for k, v in per.items()) + ' per call')
    print(f'{label}: data gradients {fl / 1e9:.1f} GFLOP in {dg:.1f} us -> {fl / dg / 1e6:.0f} TFLOP/s')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--skip-full', action='store_true')
    ap.add_argument('--kernel-only', action='store_true', help='(child process) profile the new kernels alone')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('camera_grad_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    shapes = [('small', P.SMALL, 64, 8)] + ([] if a.skip_full else [('full', P.FULL_3DIM, 128, 4)])
    if a.kernel_only:
        for label, cfg, S, B in shapes:
            kernels_alone(label, cfg, S, B, a.reps)
        return
    print(card())
    for label, cfg, S, B in shapes:
        end_to_end(label, cfg, S, B, a.reps, a.rounds)
    cmd = [sys.executable, os.path.abspath(__file__), '--kernel-only', '--reps', str(a.reps)] + (['--skip-full'] if a.skip_full else [])
    sys.stdout.flush()
    subprocess.run(cmd, check=True, env=dict(os.environ, XUNET_NO_PDL='1'))


if __name__ == '__main__':
    main()
