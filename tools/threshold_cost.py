"""Cost of dynamic thresholding (Sampler(dynamic_threshold=p), xunet_sampler_step_dynamic) against the fixed clip.

1. The step kernel alone: a CUDA graph of --launches step launches (so host launch overhead is not timed), replayed and
   timed with CUDA events, static and dynamic (p = 0.995) alternated every round, at (B, S) in (1, 64), (8, 64), (1, 128),
   (4, 128), (8, 256); both the single-step (ddim row) and the multistep (dpmpp_2m row) forms.  Median µs per launch.
2. Whole samples: views/s of `ddpm` at 256 steps, `ddim` at 50 and `dpmpp_2m` at 25 with and without thresholding, classifier-
   free guidance w = 3, CUDA-graph replay, the six samplers alternated in one process (order flipped every round), median
   over --rounds: small model at 64² with 1 and 8 views, full model at 128² with 1 and 4 views.
The card name and power limit are printed first.

    python tools/threshold_cost.py [--rounds 3] [--launches 100] [--skip-full]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from novel_view_synthesis_3d_b200.sampling import Schedule, sampler_table
from oracle import xunet_ref as R
from tools.ema_step_cost import card

P_DYN = 0.995
METHODS = (('ddpm', 256), ('ddim', 50), ('dpmpp_2m', 25))
KERNEL_SHAPES = ((1, 64), (8, 64), (1, 128), (4, 128), (8, 256))


def kernel_alone(launches, rounds):
    lib = _lib.load()
    rows = {'single-step': (sampler_table(Schedule(50), 'ddim')[0], 10),
            'multistep': (sampler_table(Schedule(25, spacing='logsnr'), 'dpmpp_2m')[0], 5)}
    for B, S in KERNEL_SHAPES:
        n = B * S * S * 3
        g = torch.Generator(device='cuda').manual_seed(0)
        eps2 = torch.randn(2 * n, device='cuda', generator=g)
        z0 = torch.randn(n, device='cuda', generator=g)
        next_z2, next_logsnr2 = torch.empty(2 * n, device='cuda'), torch.empty(2 * B, device='cuda')
        seed = torch.ones(1, dtype=torch.int64, device='cuda')
        for form, (tab_rows, k) in rows.items():
            tab = torch.tensor(tab_rows, dtype=torch.float32, device='cuda')
            pos = torch.full((1,), k, dtype=torch.int32, device='cuda')
            hist = torch.zeros(n, device='cuda') if form == 'multistep' else None
            z = z0.clone()
            zp, hp = z.data_ptr(), None if hist is None else hist.data_ptr()
            head = (eps2.data_ptr(), zp, None, n, 3.0, tab.data_ptr(), pos.data_ptr(), seed.data_ptr())
            tail = (next_z2.data_ptr(), next_logsnr2.data_ptr(), 2 * B, None)

            def static(st):
                t = tail[:-1] + (st,)
                if hp is None:
                    _lib.check(lib.xunet_sampler_step_table(*head, *t), 'sampler_step_table')
                else:
                    _lib.check(lib.xunet_sampler_step_multistep(*head, hp, *t), 'sampler_step_multistep')

            def dynamic(st):
                _lib.check(lib.xunet_sampler_step_dynamic(*head, hp, B, P_DYN, None, *tail[:-1], st), 'sampler_step_dynamic')

            graphs = {}
            for name, fn in (('static', static), ('dynamic', dynamic)):
                fn(torch.cuda.current_stream().cuda_stream)          # eager first launch (sets the shared-memory opt-in)
                torch.cuda.synchronize()
                gr = torch.cuda.CUDAGraph()
                s = torch.cuda.Stream()
                with torch.cuda.graph(gr, stream=s):
                    for _ in range(launches):
                        fn(s.cuda_stream)
                graphs[name] = gr
            times = {k2: [] for k2 in graphs}
            keys = list(graphs)
            for r in range(rounds):
                for k2 in (keys if r % 2 == 0 else keys[::-1]):
                    z.copy_(z0)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    graphs[k2].replay()
                    b.record()
                    torch.cuda.synchronize()
                    times[k2].append(a.elapsed_time(b) * 1e3 / launches)
            ms = {k2: float(np.median(v)) for k2, v in times.items()}
            print(f'kernel B={B} S={S:3d} {form:11s}: static {ms["static"]:7.2f} µs, dynamic {ms["dynamic"]:7.2f} µs '
                  f'per launch (min {min(times["dynamic"]):.2f}, max {max(times["dynamic"]):.2f})', flush=True)
            del graphs


def samples(label, model, S, views, rounds):
    params = P.create_train_state(0, 1, 1e-4, 1, S, model=model, init_on_device=label == 'full').params
    for B in views:
        batch = {k: v.numpy().astype(np.float32) for k, v in R.synthetic_batch(B, S, seed=1234)[0].items()}
        samplers = {(m, p): P.Sampler(model, params, B, S, steps=n, w=3.0, method=m, dynamic_threshold=p)
                    for m, n in METHODS for p in (None, P_DYN)}
        for s in samplers.values():
            s.capture(batch)
        torch.cuda.synchronize()
        times = {k: [] for k in samplers}
        keys = list(samplers)
        for r in range(rounds):
            for k in (keys if r % 2 == 0 else keys[::-1]):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                samplers[k].sample(batch, seed=r)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e-3)
        for (m, n) in METHODS:
            t = {p: float(np.median(times[(m, p)])) for p in (None, P_DYN)}
            f = len(samplers[(m, None)].sched)
            print(f'{label} {S}x{S} views={B} {m:9s} steps={n:3d} forwards={f:3d}: '
                  f'static {B / t[None]:7.3f} views/s {t[None] / f * 1e3:6.2f} ms/step, '
                  f'dynamic {B / t[P_DYN]:7.3f} views/s {t[P_DYN] / f * 1e3:6.2f} ms/step '
                  f'({(t[P_DYN] / t[None] - 1) * 100:+.2f} %)', flush=True)
        del samplers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--launches', type=int, default=100)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('threshold_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card())
    kernel_alone(a.launches, max(a.rounds, 5))
    samples('small', P.XUNet(dtype='bf16'), 64, (1, 8), a.rounds)
    if not a.skip_full:
        samples('full', P.XUNet.from_config(P.XUNetConfig(**{**P.FULL_3DIM.__dict__, 'dtype': 'bf16'})), 128, (1, 4), a.rounds)


if __name__ == '__main__':
    main()
