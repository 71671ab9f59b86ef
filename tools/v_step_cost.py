"""Cost of v-prediction in the training step: TrainStep(data=DeviceScenes) of a state built with prediction='eps' against one
built with prediction='v', both with loss='mse', on the small 64² model at B = 8.  The v step writes its target in the batch
kernel that writes the eps target (xunet_srn_batch_v), so the two steps run the same launches; the expected difference is
nil.  Alternated in one process (CUDA events over --steps steps per arm, median of --rounds rounds), then the batch kernel
alone of each, in µs per launch from a replayed CUDA graph of --kernel-reps launches.  The card name and power limit are
printed first.

    python tools/v_step_cost.py [--instances 40] [--views 20] [--steps 40] [--rounds 7]
"""
import argparse
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.srn_data import DeviceScenes
from tools.data_step_cost import kernel_alone, write_tree
from tools.ema_step_cost import card, time_alternating


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--instances', type=int, default=40)
    ap.add_argument('--views', type=int, default=20)
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--kernel-reps', type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'this measurement needs a CUDA device'
    print(card())
    S, B = 64, 8
    with tempfile.TemporaryDirectory() as tmp:
        write_tree(tmp, a.instances, a.views, S)
        store = DeviceScenes(tmp, S)
        steps = {}
        for pred in ('eps', 'v'):
            # one model object per arm: each state gets its own engine, so the two captured graphs do not share buffers
            st = P.create_train_state(0, 1, 1e-4, B, S, model=P.XUNet.from_config(P.SMALL), loss='mse', prediction=pred)
            steps[pred] = P.TrainStep(st, data=store, min_snr_gamma=5.0)
        fns = {pred: (lambda s=s: s()) for pred, s in steps.items()}
        for f in fns.values():
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        t = time_alternating(fns, a.steps, a.rounds)
        base = t['eps'][0]
        print(f'small 64², B={B}, loss=mse, min_snr_gamma=5, {a.steps} steps x {a.rounds} rounds per arm '
              f'(median [min, max] ms per step)')
        for key, (med, lo, hi) in t.items():
            print(f'  {key:4s} {med:8.3f} ms [{lo:.3f}, {hi:.3f}]   {100 * (med - base) / base:+.2f} % vs eps')
        for key, s in steps.items():
            us = kernel_alone(s, a.kernel_reps, a.rounds)
            print(f'  batch kernel alone ({key}): {us[0]:.2f} us per launch [{us[1]:.2f}, {us[2]:.2f}]')


if __name__ == '__main__':
    main()
