"""Training throughput from an SRN tree: the host loader against the device-resident store (TrainStep(data=DeviceScenes)).

Writes a synthetic SRN-shaped tree to a temporary directory (--instances x --views PNGs of --native² pixels, each a noise disc on
a white background, with poses and intrinsics), then, for the small 64² model at B = 8 and the full 128² model at B = 4,
alternates in one process (CUDA events over --steps steps per arm, median of --rounds rounds):
  host     : what examples/train_srn.py does by default -- SRNScenes.batches (one decoding thread) + ForwardDiffusion + TrainStep
  data     : TrainStep(data=DeviceScenes): the batch is drawn, gathered and noised by one kernel inside the step's graph
  ceiling  : TrainStep on inputs already in device memory (no loader at all)
and times the batch kernel alone, in µs per launch, from a replayed CUDA graph of --kernel-reps launches.  The card name and
power limit are printed first.

    python tools/data_step_cost.py [--instances 100] [--views 50] [--steps 40] [--rounds 5] [--skip-full]
"""
import argparse
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.srn_data import DeviceScenes, SRNScenes
from tools.ema_step_cost import card, time_alternating


def write_tree(root, instances, views, side, seed=0):
    import cv2
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[:side, :side]
    disc = (yy - side / 2) ** 2 + (xx - side / 2) ** 2 < (0.35 * side) ** 2
    for i in range(instances):
        d = os.path.join(root, f'{i:05d}')
        os.makedirs(os.path.join(d, 'rgb'))
        os.makedirs(os.path.join(d, 'pose'))
        with open(os.path.join(d, 'intrinsics.txt'), 'w') as fh:
            fh.write(f'{1.025 * side:.4f} {side / 2:.1f} {side / 2:.1f} 0.\n0. 0. 0.\n1.\n{side} {side}\n')
        for v in range(views):
            img = np.full((side, side, 3), 255, np.uint8)
            img[disc] = rng.randint(0, 256, (int(disc.sum()), 3))
            cv2.imwrite(os.path.join(d, 'rgb', f'{v:06d}.png'), img)
            q, _ = np.linalg.qr(rng.randn(3, 3))
            pose = np.eye(4)
            pose[:3, :3], pose[:3, 3] = q, 1.3 * rng.randn(3)
            with open(os.path.join(d, 'pose', f'{v:06d}.txt'), 'w') as fh:
                fh.write(' '.join(f'{x:.6f}' for x in pose.reshape(-1)) + '\n')


def kernel_alone(step, reps, rounds):
    """µs per launch of the batch kernel (slot 0 of `step`), from a replayed graph of `reps` launches."""
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        step._draw(0)
        s.synchronize()
        with torch.cuda.graph(g, stream=s):
            for _ in range(reps):
                step._draw(0)
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) * 1e3 / reps)
    return float(np.median(out)), float(min(out)), float(max(out))


def run(label, cfg, S, B, tree, steps, rounds, kernel_reps, init_on_device):
    model = P.XUNet.from_config(cfg)
    st = P.create_train_state(0, 1, 1e-4, B, S, model=model, init_on_device=init_on_device)
    t0 = time.perf_counter()
    store = DeviceScenes(tree, S, max_observations_per_instance=50)
    t_decode = time.perf_counter() - t0
    print(f'{label}: store of {store.n_items} views at {S}x{S} ({store.storage}, {store.nbytes / 2**20:.1f} MiB) built in '
          f'{t_decode:.1f} s')
    # the three arms train views of one state (only their time matters here); they share the engine and its input slots
    data_step = P.TrainStep(st, data=store)
    host_step = P.TrainStep(st)
    ds = SRNScenes(tree, img_sidelength=S, max_observations_per_instance=50, seed=0)
    fd = P.ForwardDiffusion(host_step.eng)
    stream = ds.batches(B)
    it = [0]

    def host():                                     # examples/train_srn.py's loop body at grad_accum_steps = 1
        b = next(stream)
        fd.sample(b['target'], seed=it[0])
        it[0] += 1
        dev = host_step.eng.inp
        batch = {key: b[key] for key in ('x', 'R1', 't1', 'R2', 't2', 'K')}
        batch.update({key: dev[key] for key in ('z', 'logsnr')})
        host_step(batch, dev['noise'], cond_mask=dev['cond_mask'])

    g = torch.Generator().manual_seed(1)
    dbatch = {key: torch.randn((B,) + shp, generator=g).cuda() for key, shp in
              (('x', (S, S, 3)), ('z', (S, S, 3)), ('logsnr', ()), ('R1', (3, 3)), ('t1', (3,)), ('R2', (3, 3)),
               ('t2', (3,)), ('K', (3, 3)))}
    dnoise, dmask = torch.randn(B, S, S, 3, generator=g).cuda(), torch.ones(B).cuda()
    fns = {'host': host, 'data': lambda: data_step(), 'ceiling': lambda: host_step(dbatch, dnoise, cond_mask=dmask)}
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    assert data_step.h2d_bytes == 0
    t = time_alternating(fns, steps, rounds)
    k_us = kernel_alone(data_step, kernel_reps, rounds)
    ceil = t['ceiling'][0]
    print(f'  {st.params.flat.numel()} parameters, B={B}, {cfg.dtype}, {steps} steps x {rounds} rounds per arm '
          f'(median [min, max] ms per step, images/s of the median)')
    for key, (med, lo, hi) in t.items():
        rel = '' if key == 'ceiling' else f'   {100 * (med - ceil) / ceil:+.2f} % vs ceiling'
        print(f'  {key:8s} {med:8.3f} ms [{lo:.3f}, {hi:.3f}]  {B / med * 1e3:8.1f} images/s{rel}')
    print(f'  batch kernel alone: {k_us[0]:.2f} us per launch [{k_us[1]:.2f}, {k_us[2]:.2f}] '
          f'= {100 * k_us[0] * 1e-3 / t["data"][0]:.2f} % of the data= step')
    del stream


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--instances', type=int, default=100)
    ap.add_argument('--views', type=int, default=50)
    ap.add_argument('--native', type=int, default=128)
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--kernel-reps', type=int, default=200)
    ap.add_argument('--skip-full', action='store_true')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'this measurement needs a CUDA device'
    print(card())
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        write_tree(tmp, a.instances, a.views, a.native)
        print(f'synthetic tree: {a.instances} x {a.views} views of {a.native}² PNG, written in {time.perf_counter() - t0:.1f} s')
        run('small 64²', P.SMALL, 64, 8, tmp, a.steps, a.rounds, a.kernel_reps, False)
        if not a.skip_full:
            run('full 128²', P.FULL_3DIM, 128, 4, tmp, max(8, a.steps // 4), a.rounds, a.kernel_reps, True)


if __name__ == '__main__':
    main()
