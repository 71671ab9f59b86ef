"""Cost of autoguidance (`Sampler(guide_params=...)`, `xunet_sampler_step_guide`) against classifier-free guidance.

Classifier-free guidance runs one 2B-row forward per step ([cond ; uncond]); autoguidance runs two B-row forwards, the
main model's and the guide's.  This measures which costs more, for
  cfg        one 2B-row forward of the model;
  ag-same    the model's B-row forward and a B-row forward of a guide of the same config;
  ag-half    the model's B-row forward and a B-row forward of a guide of half the width (ch and emb_ch halved; not
             buildable for the small model, whose ch = 32 is GroupNorm's minimum).

Forward: ms of each setting's forwards, one captured graph each (the 2B forward, or the two B forwards), replayed --reps
times per round, the settings alternated (order flipped each round), median [min, max] of --rounds rounds.

Sampling: views/s of the three samplers for `dpmpp_2m` at 25 steps and `ddpm` at 256, alternated per round (CUDA events
around one full `sample()`, median of --rounds).

Small 64² with 8 views in flight and full 3DiM 128² with 4.  The networks are freshly initialised: these are costs, not
image quality.  The card name and power limit are printed first and last.

    python tools/autoguide_cost.py [--reps 20] [--rounds 3] [--skip-small] [--skip-full]
"""
import argparse
import gc
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.xunet import Engine
from oracle import xunet_ref as R
from tools.ema_step_cost import card


def configs(skip_small, skip_full):
    out = [] if skip_small else [('small', P.SMALL, 64, 8)]
    if not skip_full:
        out.append(('full', P.XUNetConfig(**{**P.FULL_3DIM.__dict__, 'dtype': 'bf16'}), 128, 4))
    return out


def half_width(cfg):
    """cfg with ch and emb_ch halved, or None when the half width is not a multiple of GroupNorm's 32 groups."""
    if cfg.ch % 64:
        return None
    return P.XUNetConfig(**{**cfg.__dict__, 'ch': cfg.ch // 2, 'emb_ch': cfg.emb_ch // 2})


def guides(model, cfg, S):
    """{name: (guide XUNet, guide params)} for the autoguided settings; the params are fresh initialisations."""
    out = {'ag-same': (model, P.create_train_state(1, 1, 1e-4, 1, S, model=model, init_on_device=True).params)}
    hcfg = half_width(cfg)
    if hcfg is not None:
        half = P.XUNet.from_config(hcfg)
        out['ag-half'] = (half, P.create_train_state(2, 1, 1e-4, 1, S, model=half, init_on_device=True).params)
    return out


def time_graphs(graphs: dict, reps: int, rounds: int) -> dict:
    times = {k: [] for k in graphs}
    keys = list(graphs)
    for r in range(rounds):
        for k in (keys if r % 2 == 0 else keys[::-1]):
            graphs[k].replay()                       # one untimed replay per setting and round
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                graphs[k].replay()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / reps)
    return times


def forward_cost(label, model, params, gd, S, views, a):
    """ms of the forwards of one step of each setting."""
    batch = {k: v.numpy().astype(np.float32) for k, v in R.synthetic_batch(2 * views, S, seed=1234)[0].items()}
    cfg_eng = model.engine(2 * views, S, False)
    cfg_eng.load_inputs(batch, cond_mask=np.concatenate([np.ones(views), np.zeros(views)]).astype(np.float32))
    main = model.engine(views, S, False)
    main.load_inputs({k: v[:views] for k, v in batch.items()}, cond_mask=np.ones(views, np.float32))
    flat = model.flat_from_tree(params, S, 2 * views)
    steps = {'cfg': [lambda: cfg_eng.forward(flat, train=False)]}
    keep = []
    for name, (gm, gp) in gd.items():
        ge = Engine(gm.config, views, S, False, main.device)
        gflat = gm.flat_from_tree(gp, S, 1)
        keep.append((ge, gflat))
        steps[name] = [lambda: main.forward(flat, train=False),
                       lambda ge=ge, gflat=gflat: ge.forward(gflat, train=False, batch=main.cbatch)]
    st = torch.cuda.Stream()
    graphs = {}
    for name, fns in steps.items():
        for f in fns:
            f()                                      # every kernel runs once before the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for f in fns:
                f()
        graphs[name] = g
    torch.cuda.synchronize()
    times = time_graphs(graphs, a.reps, a.rounds)
    base = float(np.median(times['cfg']))
    print(f'forward {label} {S}², {views} views in flight, {a.reps} replays x {a.rounds} rounds (median [min, max] ms of '
          f'the forwards of one step)', flush=True)
    for name in graphs:
        t = float(np.median(times[name]))
        rows = f'1 x {2 * views} rows' if name == 'cfg' else f'2 x {views} rows'
        print(f'  {name:8s} {rows:12s} {t:8.3f} ms [{min(times[name]):.3f}, {max(times[name]):.3f}]  {t / base:5.3f} x cfg',
              flush=True)
    del graphs, keep


def sample_cost(label, model, params, gd, S, views, a):
    batch = {k: v.numpy().astype(np.float32) for k, v in R.synthetic_batch(views, S, seed=1234)[0].items()}
    for method, steps in (('dpmpp_2m', 25), ('ddpm', 256)):
        samplers = {'cfg': P.Sampler(model, params, views, S, w=3.0, steps=steps, method=method)}
        for name, (gm, gp) in gd.items():
            samplers[name] = P.Sampler(model, params, views, S, w=3.0, steps=steps, method=method, guide_params=gp,
                                       guide_model=gm)
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
        t_cfg = float(np.median(times['cfg']))
        for name, s in samplers.items():
            t = float(np.median(times[name]))
            print(f'sample {label} {S}² views={views} {method:8s} {steps:3d} steps ({len(s.sched):3d} forwards) {name:8s}: '
                  f'{views / t:8.3f} views/s  {t / len(s.sched) * 1e3:7.2f} ms/step  (min {min(times[name]):.3f} s, '
                  f'max {max(times[name]):.3f} s)  {t / t_cfg:5.3f} x cfg time', flush=True)
        del samplers
        gc.collect()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--skip-small', action='store_true')
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('autoguide_cost.py needs a CUDA device')
    torch.cuda.set_device(0)
    print(card(), flush=True)
    for label, cfg, S, views in configs(a.skip_small, a.skip_full):
        model = P.XUNet.from_config(cfg)
        params = P.create_train_state(0, 1, 1e-4, 1, S, model=model, init_on_device=True).params
        gd = guides(model, cfg, S)
        if 'ag-half' not in gd:
            print(f'{label}: ch = {cfg.ch}; a half-width guide would have ch = {cfg.ch // 2}, not a multiple of GroupNorm\'s '
                  f'32 groups: ag-half skipped', flush=True)
        forward_cost(label, model, params, gd, S, views, a)
        sample_cost(label, model, params, gd, S, views, a)
        del model, params, gd
        gc.collect()
        torch.cuda.empty_cache()
    print(card(), flush=True)


if __name__ == '__main__':
    main()
