"""Cost of the image-metric kernel (xunet_image_metrics): CUDA events around --reps launches per round on fixed SRN-like
(B, S, S, 3) pairs after warm-up, median / min / max over --rounds rounds, for each requested (B, S).  The card name and power
limit are printed first.

    python tools/metrics_cost.py [--shapes 64x128,1x128,8x256] [--reps 200] [--rounds 5]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from tests.ssim_ref import make_pair
from tools.ema_step_cost import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default='64x128,1x128,8x256', help='comma-separated BxS')
    ap.add_argument('--reps', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('metrics_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    for shape in a.shapes.split(','):
        B, S = map(int, shape.split('x'))
        p, t = (torch.as_tensor(x).cuda() for x in make_pair('srn', B, S, seed=1))
        for _ in range(10):
            P.image_metrics(p, t)
        torch.cuda.synchronize()
        times = []
        for _ in range(a.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                P.image_metrics(p, t)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) / a.reps)
        med = float(np.median(times))
        print(f'B={B} S={S}: {1e3 * med:.1f} us per call (min {1e3 * min(times):.1f}, max {1e3 * max(times):.1f}), '
              f'{1e3 * med / B:.2f} us per image, {a.reps} calls x {a.rounds} rounds')


if __name__ == '__main__':
    main()
