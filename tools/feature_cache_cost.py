"""Cost of the sampler feature cache (DeepCache, `xunet_set_feature_cache`, `Sampler(cache_interval=N, cache_level=L)`).

Forward: ms of one full forward and of one cheap forward at every legal level L, each a captured graph of the guided
sampler's 2B-batch forward replayed --reps times per round, the settings alternated (order flipped each round), median
[min, max] of --rounds rounds; the kernel count of each (`xunet_count_kernels` at that level); and the share of the
forward's conv and attention FLOPs the cheap forward recomputes, from the plan's launch shapes, next to its measured time
share.

Sampling: views/s of `Sampler` with cache_interval N in {1, 2, 3, 5} at L = 1, for `ddpm` at 256 steps and `dpmpp_2m` at
25, alternated per round (CUDA events around one full `sample()`, median of --rounds).

Small 64² with 8 views in flight (a 16-row engine) and full 3DiM 128² with 4 (8 rows).  The networks are freshly
initialised: these are costs, not image quality.  The card name and power limit are printed first and last.

    python tools/feature_cache_cost.py [--reps 20] [--rounds 3] [--intervals 1,2,3,5] [--skip-small] [--skip-full]
"""
import argparse
import ctypes as C
import gc
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import _lib
from oracle import xunet_ref as R
from tests.feature_cache_ref import kept_blocks        # which parameter blocks a cheap forward at L reads
from tests.util import to_ref_cfg
from tools.ema_step_cost import card


def configs(skip_small, skip_full):
    out = [] if skip_small else [('small', P.SMALL, 64, 8)]
    if not skip_full:
        out.append(('full', P.XUNetConfig(**{**P.FULL_3DIM.__dict__, 'dtype': 'bf16'}), 128, 4))
    return out


def flop_share(lib, eng, rcfg, level):
    """FLOPs of the conv and attention launches a cheap forward at `level` runs, over those of the full forward: a conv is
    2 N Ho Wo Co Ci k², an attention 4 N L² C (scores and the weighted sum, L tokens a frame); an attention launch belongs
    to the block of the conv launch before it (its qkv projection)."""
    names = list(eng.spec)
    kept = kept_blocks(rcfg, level)
    info = _lib.XunetLaunchInfo()
    total = keep = 0.0
    owner = None
    for i in range(lib.xunet_plan_launch_count(eng.h)):
        assert lib.xunet_plan_launch(eng.h, i, C.byref(info)) == 0
        if info.kind == _lib.LAUNCH_CONV:
            leaf = names[info.leaf].split('/')
            owner = '/'.join(leaf[:2]) if leaf[0] == 'ConditioningProcessor_0' else leaf[0]
            f = 2.0 * info.N * info.Ho * info.Wo * info.Co * info.Ci * info.ksize ** 2
        else:
            f = 4.0 * info.N * info.L ** 2 * info.C
        total += f
        keep += f if owner in kept else 0.0
    return keep / total


def forward_cost(lib, label, cfg, S, views, a):
    model = P.XUNet.from_config(cfg)
    rcfg = to_ref_cfg(model.config)
    params = P.create_train_state(0, 1, 1e-4, 1, S, model=model, init_on_device=True).params
    B = 2 * views                                    # the guided sampler's [cond ; uncond] batch
    eng = model.engine(B, S, False)
    flat = model.flat_from_tree(params, S, B)
    batch = {k: v.numpy().astype(np.float32) for k, v in R.synthetic_batch(B, S, seed=1234)[0].items()}
    eng.load_inputs(batch, cond_mask=np.concatenate([np.ones(views), np.zeros(views)]).astype(np.float32))
    levels = list(range(len(cfg.ch_mult)))
    graphs, kernels = {}, {}
    st = torch.cuda.Stream()
    for lvl in levels:
        _lib.check(lib.xunet_set_feature_cache(eng.h, 0), 'set_feature_cache')
        eng.forward(flat, train=False)               # a full forward leaves the cached tensors
        _lib.check(lib.xunet_set_feature_cache(eng.h, lvl), 'set_feature_cache')
        kernels[lvl] = eng.count_kernels(flat)[0]
        eng.forward(flat, train=False)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            eng.forward(flat, train=False)
        graphs[lvl] = g
    _lib.check(lib.xunet_set_feature_cache(eng.h, 0), 'set_feature_cache')
    torch.cuda.synchronize()
    times = {lvl: [] for lvl in levels}
    for r in range(a.rounds):
        for lvl in (levels if r % 2 == 0 else levels[::-1]):
            graphs[lvl].replay()                     # one untimed replay per setting and round
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                graphs[lvl].replay()
            e1.record()
            e1.synchronize()
            times[lvl].append(e0.elapsed_time(e1) / a.reps)
    base = float(np.median(times[0]))
    print(f'forward {label} {S}², {views} views in flight ({B}-row engine), {a.reps} replays x {a.rounds} rounds '
          f'(median [min, max] ms per forward)', flush=True)
    for lvl in levels:
        t = float(np.median(times[lvl]))
        share = 1.0 if lvl == 0 else flop_share(lib, eng, rcfg, lvl)
        print(f'  {"full" if lvl == 0 else f"cheap L={lvl}":11s} {t:8.3f} ms [{min(times[lvl]):.3f}, {max(times[lvl]):.3f}]  '
              f'kernels {kernels[lvl]:4d}  time share {t / base:.3f}  FLOP share {share:.3f}', flush=True)
    del graphs, eng, flat
    return model, params


def sample_cost(model, params, label, S, views, a):
    batch = {k: v.numpy().astype(np.float32) for k, v in R.synthetic_batch(views, S, seed=1234)[0].items()}
    samplers = {}
    for method, steps in (('ddpm', 256), ('dpmpp_2m', 25)):
        for n in a.intervals:
            samplers[(method, steps, n)] = P.Sampler(model, params, views, S, w=3.0, steps=steps, method=method,
                                                     cache_interval=n, cache_level=1)
    for s in samplers.values():
        s.capture(batch)
        s.sample(batch, seed=0, _max_steps=max(a.intervals) + 1)   # every graph (full and cheap) captured
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
    for (method, steps, n), s in samplers.items():
        t = float(np.median(times[(method, steps, n)]))
        t1 = float(np.median(times[(method, steps, a.intervals[0])]))
        print(f'sample {label} {S}² views={views} {method:8s} {steps:3d} steps ({len(s.sched):3d} forwards) N={n} L=1: '
              f'{views / t:8.3f} views/s  {t / len(s.sched) * 1e3:6.2f} ms/step  (min {min(times[(method, steps, n)]):.3f} s, '
              f'max {max(times[(method, steps, n)]):.3f} s)  {t1 / t:5.2f} x N={a.intervals[0]}', flush=True)
    del samplers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--intervals', default='1,2,3,5', help='cache intervals N to sample with (the first is the baseline)')
    ap.add_argument('--skip-small', action='store_true')
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    a.intervals = [int(x) for x in a.intervals.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('feature_cache_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    lib = _lib.load()
    print(card(), flush=True)
    for label, cfg, S, views in configs(a.skip_small, a.skip_full):
        model, params = forward_cost(lib, label, cfg, S, views, a)
        sample_cost(model, params, label, S, views, a)
        del model, params
        gc.collect()
        torch.cuda.empty_cache()
    print(card(), flush=True)


if __name__ == '__main__':
    main()
