"""Cost of the consistency score's grid fit (consistency.fit_field): G = 128, 40 views at 128^2 of the analytic sphere scene of
tests/test_gpu_field.py, the default iterations and rays.  Device events around whole fits after a warm-up fit, median / min /
max over --rounds rounds; then ms per iteration, rays/s and one render of the 40 views.  The card name and power limit are
printed first.

    python tools/field_cost.py [--grid 128] [--side 128] [--views 40] [--iters N] [--rays N] [--rounds 3]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from novel_view_synthesis_3d_b200 import consistency as CS
from tests.test_field_cpu import cameras
from tests.test_gpu_field import SPHERES, sphere_grid
from tools.ema_step_cost import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--grid', type=int, default=128)
    ap.add_argument('--side', type=int, default=128)
    ap.add_argument('--views', type=int, default=40)
    ap.add_argument('--iters', type=int, default=CS.ITERS)
    ap.add_argument('--rays', type=int, default=CS.RAYS)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('field_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    G, S = a.grid, a.side
    R, t, K = cameras(a.views, S, seed=0)
    b = CS.default_bound(t)
    scene = CS.Field(grid=sphere_grid(G, b, SPHERES).contiguous(), bound=b, step=b / (G - 1), near=0.0, background=1.0, S=S,
                     loss=None)
    views = scene.render(R, t, K)
    CS.fit_field(views, R, t, K, grid=G, iters=20, rays=a.rays)          # warm-up: module load, graph capture
    torch.cuda.synchronize()
    times, f = [], None
    for _ in range(a.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f = CS.fit_field(views, R, t, K, grid=G, iters=a.iters, rays=a.rays)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    med = float(np.median(times))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = f.render(R, t, K)
    e1.record()
    e1.synchronize()
    mse = float(((out - views) ** 2).mean() / 4)
    print(f'G={G} views={a.views}x{S}^2 iters={a.iters} rays={a.rays}: fit {med / 1e3:.3f} s (min {min(times) / 1e3:.3f}, '
          f'max {max(times) / 1e3:.3f}, {a.rounds} rounds), {1e3 * med / a.iters:.1f} us per iteration, '
          f'{a.iters * a.rays / (med / 1e3) / 1e6:.1f} M rays/s; render of the {a.views} views {e0.elapsed_time(e1):.2f} ms; '
          f'final data loss {f.loss[-1].item():.3e}, fitted-view PSNR {-10 * np.log10(mse):.2f} dB')


if __name__ == '__main__':
    main()
