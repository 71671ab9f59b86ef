"""Cost of the weight EMA fused into the Adam kernel: TrainStep with and without EMA in one process, alternated over several
rounds (CUDA events over >= 20 graph replays after warm-up), and the Adam launch alone through the C-ABI at the full-model
parameter count, with achieved HBM bandwidth against the bytes the kernel must move.

    python tools/ema_step_cost.py [--steps 20] [--rounds 5] [--skip-full]
"""
import argparse
import os
import subprocess
import sys
from dataclasses import replace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from bench import make_host_batches

N_FULL = 438831363                          # FULL_3DIM at 128x128
BYTES_ADAM, BYTES_EMA = 28, 8               # per parameter: p,m,v read+written, g read;  ema read+written


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:
        q = f'nvidia-smi unavailable ({e})'
    return f'{name}, power limit / max SM clock: {q}'


def time_alternating(fns: dict, reps: int, rounds: int):
    """Median ms per call of each fn, the fns alternated within every round (order flipped each round)."""
    out = {k: [] for k in fns}
    keys = list(fns)
    for r in range(rounds):
        for k in (keys if r % 2 == 0 else keys[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fns[k]()
            b.record()
            torch.cuda.synchronize()
            out[k].append(a.elapsed_time(b) / reps)
    return {k: (float(np.median(v)), float(min(v)), float(max(v))) for k, v in out.items()}


def adam_alone(reps, rounds):
    lib = _lib.load()
    n = N_FULL
    p, g, m, v, e = (torch.randn(n, device='cuda') * 1e-2 for _ in range(5))
    st = torch.cuda.current_stream().cuda_stream
    fns = {
        'adam': lambda: _lib.check(lib.xunet_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, 1, None, 1e-4,
                                                       0.9, 0.999, 1e-8, 1.0, st)),
        'adam+ema': lambda: _lib.check(lib.xunet_adam_ema_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(),
                                                               e.data_ptr(), n, 1, None, 1e-4, 0.9, 0.999, 1e-8, 1.0, 0.9999, st)),
    }
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    del p, g, m, v, e
    torch.cuda.empty_cache()
    ta, te = t['adam'][0], t['adam+ema'][0]
    print(f'Adam launch alone, n = {n} parameters:')
    print(f'  adam      {ta:8.3f} ms  (min {t["adam"][1]:.3f}, max {t["adam"][2]:.3f})  '
          f'{BYTES_ADAM * n / ta / 1e6:7.0f} GB/s over {BYTES_ADAM} B/param')
    print(f'  adam+ema  {te:8.3f} ms  (min {t["adam+ema"][1]:.3f}, max {t["adam+ema"][2]:.3f})  '
          f'{(BYTES_ADAM + BYTES_EMA) * n / te / 1e6:7.0f} GB/s over {BYTES_ADAM + BYTES_EMA} B/param')
    print(f'  EMA share {te - ta:8.3f} ms  (a separate pass would move 12 B/param = {12 * n / 1e9:.2f} GB, '
          f'>= {12 * n / 3.35e12 * 1e3:.2f} ms at the 3.35 TB/s data-sheet rate)')


def train_step(label, cfg, S, B, reps, rounds, init_on_device):
    """One model and one set of buffers; two TrainStep views of them, one with the EMA buffer and one without.  Both train
    the same weights (the numbers they compute are irrelevant here; only the time is)."""
    model = P.XUNet.from_config(cfg)
    st_ema = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=init_on_device, ema_decay=0.9999)
    st_plain = replace(st_ema, ema_params=None, ema_decay=None, opt_state=replace(st_ema.opt_state))
    steps = {'no EMA': P.TrainStep(st_plain), 'EMA': P.TrainStep(st_ema)}
    (batch, noise), = make_host_batches(1, B, S, 1234)
    cond = np.ones(B, np.float32)
    fns = {k: (lambda s=s: s(batch, noise, cond_mask=cond)) for k, s in steps.items()}
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = time_alternating(fns, reps, rounds)
    n = st_ema.params.flat.numel()
    a, e = t['no EMA'][0], t['EMA'][0]
    print(f'{label}: {n} parameters, B={B}, {S}x{S}, {cfg.dtype}, {reps} steps x {rounds} rounds per arm')
    for k, (med, lo, hi) in t.items():
        print(f'  {k:7s} {med:9.3f} ms/step  (min {lo:.3f}, max {hi:.3f})')
    print(f'  EMA cost {e - a:+.3f} ms/step = {100 * (e - a) / a:+.2f} %  '
          f'(bytes added: {BYTES_EMA * n / 1e9:.3f} GB, >= {BYTES_EMA * n / 3.35e12 * 1e3:.3f} ms at 3.35 TB/s)')
    del steps, st_plain, st_ema, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ema_step_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    adam_alone(max(a.steps, 20), a.rounds)
    train_step('small', P.SMALL, 64, 8, a.steps, a.rounds, init_on_device=False)
    if not a.skip_full:
        train_step('full', P.FULL_3DIM, 128, 4, a.steps, a.rounds, init_on_device=True)


if __name__ == '__main__':
    main()
