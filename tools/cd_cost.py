"""Cost of consistency distillation, training and sampling.

Training: ms per update of a consistency-distillation `TrainStep(data=DeviceScenes, teacher=ConsistencyTeacher(w=3))` (the
draw, one guided teacher forward of the 2B batch, the teacher step, the target forward of the student's own weights on its
training engine, the target kernel, then the student's forward and backward) against a plain v `TrainStep(data=)` and a
progressive-distillation `TrainStep(teacher=Teacher(w=3))` of the same student, small 64² B=8 and full 128² B=4, in one
process, each distillation arm alternated with the v arm (CUDA events over --steps steps per arm, median [min, max] of
--rounds rounds).

Sampling: views/s of a consistency student at K = 1, 2, 4 steps without guidance (`Sampler(method='consistency', w=None)`,
one B-batch forward per step, on `consistency_grid(256, K)`) against the guided teacher (w = 3, the 2B batch) with
DPM-Solver++(2M) at 25 steps and with the reference DDPM sampler at 256, small 64² at 1 and 8 views and full 128² at 1
and 4, alternated per round (CUDA events around one full `sample()`).

The networks are freshly initialised: these are costs, not image quality.  The card name and power limit are printed first.

    python tools/cd_cost.py [--steps 10] [--rounds 3] [--ks 1,2,4] [--skip-small] [--skip-full] [--skip-train]
"""
import argparse
import gc
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
from tools.distill_cost import TEACHER_STEPS, configs
from tools.ema_step_cost import card, time_alternating


def train_cost(label, cfg, S, B, a):
    with tempfile.TemporaryDirectory() as tmp:
        write_tree(tmp, a.instances, a.views, S)
        store = DeviceScenes(tmp, S)
        model = P.XUNet.from_config(cfg)
        st = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=True, loss='mse', prediction='v')
        print(f'train {label} {S}², B={B}: teacher DDIM grid of {TEACHER_STEPS}, w=3, {a.steps} steps x {a.rounds} rounds per '
              f'arm (median [min, max] ms per update)', flush=True)
        # each distillation arm is alternated with the plain v arm; the arms train one v / mse state on one model object
        # (one training engine, one set of parameter and Adam buffers), and one teacher lives at a time: the full model does
        # not hold two teachers' engines beside the training engine.  The values are a fresh network's either way
        for name, cls in (('pd', P.Teacher), ('cd', P.ConsistencyTeacher)):
            teacher = cls(model, st.params, TEACHER_STEPS, batch_size=B, img_sidelength=S, w=3.0)
            steps = {'v': P.TrainStep(st, data=store), name: P.TrainStep(st, data=store, teacher=teacher)}
            fns = {k: (lambda s=s: s()) for k, s in steps.items()}
            for f in fns.values():
                for _ in range(3):
                    f()
            torch.cuda.synchronize()
            t = time_alternating(fns, a.steps, a.rounds)
            base = t['v'][0]
            for k, (med, lo, hi) in t.items():
                print(f'  {k:3s} {med:9.3f} ms [{lo:.3f}, {hi:.3f}]   {med / base:.3f} x the v step   '
                      f'{B / med * 1e3:8.1f} images/s', flush=True)
            del steps, fns, f, teacher
            gc.collect()
            torch.cuda.empty_cache()
        del st, model, store
        gc.collect()
        torch.cuda.empty_cache()


def sample_cost(label, cfg, S, views, a):
    model = P.XUNet.from_config(cfg)
    params = P.create_train_state(0, 1, 1e-4, 1, S, model=model, init_on_device=True).params
    for B in views:
        batch = {k: v.numpy().astype(np.float32) for k, v in R.synthetic_batch(B, S, seed=1234)[0].items()}
        samplers = {'teacher ddpm 256 w=3': P.Sampler(model, params, B, S, w=3.0, steps=256),
                    'teacher dpmpp_2m 25 w=3': P.Sampler(model, params, B, S, w=3.0, steps=25, method='dpmpp_2m')}
        for k in a.ks:
            samplers[f'cd student K={k} w=None'] = P.Sampler(model, params, B, S, w=None, method='consistency',
                                                             prediction='v',
                                                             timesteps=P.consistency_grid(TEACHER_STEPS, k))
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
        base = {k: float(np.median(times[k])) for k in keys[:2]}
        for k, s in samplers.items():
            t = float(np.median(times[k]))
            print(f'sample {label} {S}² views={B} {k:24s} forwards={len(s.sched):3d} batch={s.eng.B:2d}: '
                  f'{B / t:9.3f} views/s, {t / len(s.sched) * 1e3:6.2f} ms/step (min {min(times[k]):.4f} s, '
                  f'max {max(times[k]):.4f} s)   {base[keys[0]] / t:7.1f} x ddpm 256, {base[keys[1]] / t:5.2f} x dpmpp_2m 25',
                  flush=True)
        del samplers
    del model, params
    gc.collect()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--instances', type=int, default=40)
    ap.add_argument('--views', type=int, default=20)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--ks', default='1,2,4', help='consistency sampling step counts K')
    ap.add_argument('--skip-small', action='store_true')
    ap.add_argument('--skip-full', action='store_true')
    ap.add_argument('--skip-train', action='store_true')
    a = ap.parse_args()
    a.ks = [int(x) for x in a.ks.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('cd_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card(), flush=True)
    for label, cfg, S, B, views in configs(a.skip_small, a.skip_full):
        if not a.skip_train:
            train_cost(label, cfg, S, B, a)
        sample_cost(label, cfg, S, views, a)


if __name__ == '__main__':
    main()
