"""Cost of progressive distillation, training and sampling.

Training: ms per update of a distillation `TrainStep(data=DeviceScenes, teacher=Teacher(w=3))` (the draw, two guided teacher
forwards of the 2B batch, the teacher step and target kernels, then the student's forward and backward) against a plain
v `TrainStep(data=DeviceScenes)` of the same student, small 64² B=8 and full 128² B=4, alternated in one process (CUDA
events over --steps steps per arm, median [min, max] of --rounds rounds).

Sampling: views/s of a student's DDIM at N steps without guidance (`Sampler(w=None)`, one B-batch forward per step) against
its teacher's DDIM at 2N steps with guidance w = 3 (the 2B batch), on the nested grids of `distill_grid`, small 64² at 1
and 8 views and full 128² at 1 and 4, alternated per round (CUDA events around one full `sample()`).

The networks are freshly initialised: these are costs, not image quality.  The card name and power limit are printed first.

    python tools/distill_cost.py [--steps 10] [--rounds 3] [--student-steps 8,32] [--skip-small] [--skip-full] [--skip-train]
"""
import argparse
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.srn_data import DeviceScenes
from oracle import xunet_ref as R
from tools.data_step_cost import write_tree
from tools.ema_step_cost import card, time_alternating

TEACHER_STEPS = 256


def configs(skip_small, skip_full):
    out = [] if skip_small else [('small', P.SMALL, 64, 8, (1, 8))]
    if not skip_full:
        out.append(('full', P.XUNetConfig(**{**P.FULL_3DIM.__dict__, 'dtype': 'bf16'}), 128, 4, (1, 4)))
    return out


def train_cost(label, cfg, S, B, a):
    with tempfile.TemporaryDirectory() as tmp:
        write_tree(tmp, a.instances, a.views, S)
        store = DeviceScenes(tmp, S)
        # both students on one model object, so one training engine (21 GB of workspace for the full model at B = 4): the
        # two captured steps run one after the other and each overwrites what it reads
        model = P.XUNet.from_config(cfg)
        st_v = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=True, loss='mse', prediction='v')
        teacher = P.Teacher(model, st_v.params, TEACHER_STEPS, batch_size=B, img_sidelength=S, w=3.0)
        st_d = P.create_distill_state(teacher, 1e-4)
        steps = {'v': P.TrainStep(st_v, data=store), 'distill': P.TrainStep(st_d, data=store, teacher=teacher)}
        fns = {k: (lambda s=s: s()) for k, s in steps.items()}
        for f in fns.values():
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        t = time_alternating(fns, a.steps, a.rounds)
        base = t['v'][0]
        print(f'train {label} {S}², B={B}: teacher DDIM grid of {len(teacher.grid)}, w=3, {a.steps} steps x {a.rounds} '
              f'rounds per arm (median [min, max] ms per update)', flush=True)
        for k, (med, lo, hi) in t.items():
            print(f'  {k:8s} {med:9.3f} ms [{lo:.3f}, {hi:.3f}]   {med / base:.3f} x the v step   {B / med * 1e3:8.1f} images/s',
                  flush=True)
        del steps, fns, st_d, st_v, teacher
        torch.cuda.empty_cache()


def sample_cost(label, cfg, S, views, a):
    model = P.XUNet.from_config(cfg)
    params = P.create_train_state(0, 1, 1e-4, 1, S, model=model, init_on_device=True).params
    for n in a.student_steps:
        rounds = int(np.log2(TEACHER_STEPS // n))
        for B in views:
            batch = {k: v.numpy().astype(np.float32) for k, v in R.synthetic_batch(B, S, seed=1234)[0].items()}
            samplers = {
                f'teacher ddim {2 * n} steps w=3': P.Sampler(model, params, B, S, w=3.0, method='ddim', prediction='v',
                                                             timesteps=P.distill_grid(TEACHER_STEPS, rounds - 1)),
                f'student ddim {n} steps w=None': P.Sampler(model, params, B, S, w=None, method='ddim', prediction='v',
                                                            timesteps=P.distill_grid(TEACHER_STEPS, rounds))}
            for s in samplers.values():
                s.capture(batch)
            torch.cuda.synchronize()
            times = {k: [] for k in samplers}
            keys = list(samplers)
            for r in range(a.rounds):
                for k in (keys if r % 2 == 0 else keys[::-1]):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    samplers[k].sample(batch, seed=r)
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1) * 1e-3)
            base = float(np.median(times[keys[0]]))
            for k, s in samplers.items():
                t = float(np.median(times[k]))
                print(f'sample {label} {S}² views={B} {k:28s} forwards={len(s.sched):3d} batch={s.eng.B:2d}: '
                      f'{B / t:8.3f} views/s, {t / len(s.sched) * 1e3:6.2f} ms/step (min {min(times[k]):.4f} s, '
                      f'max {max(times[k]):.4f} s)   {base / t:.2f} x the teacher', flush=True)
            del samplers
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--instances', type=int, default=40)
    ap.add_argument('--views', type=int, default=20)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--student-steps', default='8,32', help='student step counts N (the teacher runs 2N); powers of 2')
    ap.add_argument('--skip-small', action='store_true')
    ap.add_argument('--skip-full', action='store_true')
    ap.add_argument('--skip-train', action='store_true')
    a = ap.parse_args()
    a.student_steps = [int(x) for x in a.student_steps.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('distill_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card(), flush=True)
    for label, cfg, S, B, views in configs(a.skip_small, a.skip_full):
        if not a.skip_train:
            train_cost(label, cfg, S, B, a)
        sample_cost(label, cfg, S, views, a)


if __name__ == '__main__':
    main()
