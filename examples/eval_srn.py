"""Scores sampled views against held-out ground truth on SRN: PSNR and SSIM per view (novel_view_synthesis_3d_b200.metrics,
computed on the GPU from the sampler's output), following the single-view protocol of pixelNeRF that 3DiM reports: each
instance is conditioned on one source view (view 64 by default) and every scored target view is generated from it.

    python examples/eval_srn.py cars_test --ckpt checkpoints --prefix ema --side 128 --steps 256 --w 3 \\
        --source-view 64 --targets 10 --max-instances 20 --views-in-flight 8 --mode independent --out eval/
    python examples/eval_srn.py cars_test --ckpt checkpoints --prefix ema --side 128 --method dpmpp_2m --steps 25 --out eval_dpm/
    python examples/eval_srn.py cars_test --ckpt checkpoints --prefix ema --side 128 --method dpmpp_2m --steps 25 \\
        --dynamic-threshold 0.995 --out eval_dpm_dyn/
    python examples/eval_srn.py cars_test --ckpt checkpoints_v --prefix ema --side 128 --prediction v --method dpmpp_2m \\
        --steps 25 --out eval_v/
    python examples/eval_srn.py cars_test --ckpt checkpoints_d6 --prefix ema --side 128 --steps 256 --distilled 6 --out eval_d6/
    python examples/eval_srn.py cars_test --ckpt checkpoints_cd --prefix ema --side 128 --consistency 4 --out eval_cd4/
    python examples/eval_srn.py cars_test --ckpt checkpoints --prefix ema --side 128 --steps 256 --cache-interval 3 --out eval_dc3/
    python examples/eval_srn.py cars_test --ckpt checkpoints --prefix phema010 --guide-prefix guide005 --w 1 --side 128 \
        --method dpmpp_2m --steps 25 --out eval_ag/

Modes:
  independent  each target is sampled from the source alone (Sampler.sample, the reference's k = 1 sampler); the targets
               of one instance are batched --views-in-flight at a time.
  stochastic   3DiM's stochastic conditioning (Sampler.sample_views): the source is the pool and the targets are generated
               in order, each step conditioned on a random view of the pool (the source and the targets generated so far);
               instances are batched --views-in-flight at a time.
Writes out/metrics.jsonl (one {instance, view, psnr, ssim} line per scored view) and out/summary.json (mean PSNR, mean SSIM,
the number of views, the prediction the checkpoint was read with, the distillation round --distilled, the consistency
sampling steps --consistency and the teacher grid's N of a consistency student, the forwards per view and the arguments),
prints the summary as the last line of stdout, and with --save-views writes each generated view as out/views/<instance>_<view>.png.  Seeds derive from --seed, so equal arguments give equal files.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.srn_data import SRNScenes

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from distill_srn import cd_steps  # noqa: E402
from sample_srn import add_guide_args, load_guide  # noqa: E402


def select_targets(n_views: int, source: int, count: int) -> list:
    """The target views of an instance with n_views views: `count` views spaced evenly over the views other than `source`,
    in increasing order; all of them when count is 0 or at least their number."""
    rest = [v for v in range(n_views) if v != source]
    if count <= 0 or count >= len(rest):
        return rest
    return [rest[i] for i in np.linspace(0, len(rest), num=count, endpoint=False, dtype=int)]


def _pad(a: np.ndarray, n: int) -> np.ndarray:
    """Rows of `a` padded to n by repeating the last one (the sampler's batch is fixed; padding rows are not scored)."""
    return np.concatenate([a, np.repeat(a[-1:], n - len(a), axis=0)]) if len(a) < n else a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('folder')
    ap.add_argument('--ckpt', default='checkpoints')
    ap.add_argument('--prefix', default='model', help="checkpoint prefix: 'ema' scores the weight EMA of train_srn.py")
    ap.add_argument('--side', type=int, default=64)
    ap.add_argument('--steps', type=int, default=256)
    ap.add_argument('--w', type=float, default=3.0)
    ap.add_argument('--method', choices=P.sampling.METHODS, default='ddpm',
                    help="ddpm: the reference's ancestral sampler; ddim and dpmpp_2m (DPM-Solver++(2M)) need tens of steps")
    ap.add_argument('--eta', type=float, default=0.0, help='DDIM stochasticity in [0, 1] (0: deterministic, 1: DDPM)')
    ap.add_argument('--spacing', choices=P.sampling.SPACINGS, default=None,
                    help='timestep spacing (default: logsnr for dpmpp_2m, linear otherwise)')
    ap.add_argument('--dynamic-threshold', type=float, default=None, metavar='P',
                    help='threshold x0 per view at the P-quantile of |x0| (Imagen: 0.995) instead of clipping it to [-1, 1]')
    ap.add_argument('--prediction', choices=P.sampling.PREDICTIONS, default='eps',
                    help='what the checkpoint predicts: the noise (eps) or v (a model trained with --prediction v)')
    ap.add_argument('--distilled', type=int, default=0, metavar='R',
                    help='sample a student distilled R times (examples/distill_srn.py) from a --steps-step teacher: DDIM '
                         '(eta 0) on distill_grid(--steps, R) without guidance, reading v; --method, --eta, --spacing, --w '
                         'and --prediction are then ignored')
    ap.add_argument('--consistency', type=int, default=0, metavar='K',
                    help='sample a consistency-distilled student (examples/distill_srn.py --consistency N) in K steps: '
                         'multistep consistency sampling on consistency_grid(N, K) without guidance, reading v, with N read '
                         'from the state<step> checkpoint in --ckpt (a directory); --steps, --method, --eta, --spacing, --w '
                         'and --prediction are then ignored')
    ap.add_argument('--cache-interval', type=int, default=1, metavar='N',
                    help='feature cache (DeepCache): a full forward every N steps, and between them cheap forwards that '
                         'recompute only the levels below --cache-level and read the deeper feature of the last full one '
                         '(1: every forward full, the default)')
    ap.add_argument('--cache-level', type=int, default=1, metavar='L',
                    help='feature-cache level in [1, levels - 1]: the cheap forwards recompute the levels below L')
    add_guide_args(ap)
    ap.add_argument('--source-view', type=int, default=64, help='conditioning view of every instance (pixelNeRF / 3DiM: 64)')
    ap.add_argument('--targets', type=int, default=0, help='target views per instance, spaced evenly; 0 = all other views')
    ap.add_argument('--max-instances', type=int, default=-1, help='score the first N instances of the sorted list')
    ap.add_argument('--views-in-flight', type=int, default=8, help='sampler batch size')
    ap.add_argument('--mode', choices=('independent', 'stochastic'), default='independent')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default='eval')
    ap.add_argument('--save-views', action='store_true')
    a = ap.parse_args()
    if a.views_in_flight < 1:
        ap.error('--views-in-flight must be >= 1')
    guide = load_guide(ap, a)
    params = P.checkpoint.restore_checkpoint(a.ckpt, prefix=a.prefix)
    if params is None:
        raise FileNotFoundError('Checkpoint does not exist')
    ds = SRNScenes(a.folder, img_sidelength=a.side, max_num_instances=a.max_instances)
    insts = []
    for i in range(len(ds.instances)):
        n = len(ds.instances[i]['imgs'])
        if a.source_view < 0 or a.source_view >= n:
            raise SystemExit(f"instance {ds.instances[i]['name']} has {n} views; --source-view {a.source_view} does not exist")
        insts.append((i, select_targets(n, a.source_view, a.targets)))
    B = a.views_in_flight
    cache = dict(cache_interval=a.cache_interval, cache_level=a.cache_level)
    if a.consistency:
        sampler = P.Sampler(P.XUNet(), params, B, a.side, w=None, method='consistency', prediction='v',
                            timesteps=P.consistency_grid(cd_steps(a.ckpt), a.consistency),
                            dynamic_threshold=a.dynamic_threshold, **cache)
    elif a.distilled:
        sampler = P.Sampler(P.XUNet(), params, B, a.side, w=None, method='ddim', prediction='v',
                            timesteps=P.distill_grid(a.steps, a.distilled), dynamic_threshold=a.dynamic_threshold, **cache)
    else:
        sampler = P.Sampler(P.XUNet(), params, B, a.side, steps=a.steps, w=a.w, method=a.method, eta=a.eta,
                            spacing=a.spacing, dynamic_threshold=a.dynamic_threshold, prediction=a.prediction,
                            guide_params=guide, **cache)
    os.makedirs(a.out, exist_ok=True)
    if a.save_views:
        os.makedirs(os.path.join(a.out, 'views'), exist_ok=True)
    records = []

    def score(name, views, gen, truth):
        m = P.image_metrics(gen, truth)
        for v, psnr, ssim in zip(views, m['psnr'].tolist(), m['ssim'].tolist()):
            records.append(dict(instance=name, view=int(v), psnr=psnr, ssim=ssim))
        if a.save_views:
            for v, img in zip(views, gen.cpu().numpy()):
                P.sampling.save_view(os.path.join(a.out, 'views', f'{name}_{v:06d}.png'), img)

    if a.mode == 'independent':
        for i, targets in insts:
            d = ds.instance_views(i)
            s = a.source_view
            for c, j0 in enumerate(range(0, len(targets), B)):
                tv = targets[j0:j0 + B]
                n = len(tv)
                batch = dict(x=_pad(np.repeat(d['x'][s:s + 1], n, 0), B), R1=_pad(np.repeat(d['R'][s:s + 1], n, 0), B),
                             t1=_pad(np.repeat(d['t'][s:s + 1], n, 0), B), R2=_pad(d['R'][tv], B), t2=_pad(d['t'][tv], B),
                             K=np.repeat(d['K'][None], B, 0))
                gen = sampler.sample(batch, seed=(a.seed * 1000003 + i) * 1009 + c)
                score(d['name'], tv, gen[:n], d['x'][tv])
    else:
        # a batch holds up to B consecutive instances with the same number of targets (one row per instance)
        groups = []
        for i, targets in insts:
            if groups and len(groups[-1]) < B and len(groups[-1][0][1]) == len(targets):
                groups[-1].append((i, targets))
            else:
                groups.append([(i, targets)])
        for g in groups:
            if not g[0][1]:
                continue
            ds_g =[(ds.instance_views(i), t) for i, t in g]
            s, n = a.source_view, len(g)
            src = _pad(np.stack([d['x'][s:s + 1] for d, _ in ds_g]), B)
            poses = {'R': _pad(np.stack([d['R'][s:s + 1] for d, _ in ds_g]), B),
                     't': _pad(np.stack([d['t'][s:s + 1] for d, _ in ds_g]), B)}
            tposes = {'R': _pad(np.stack([d['R'][t] for d, t in ds_g]), B), 't': _pad(np.stack([d['t'][t] for d, t in ds_g]), B)}
            K = _pad(np.stack([d['K'] for d, _ in ds_g]), B)
            gen = sampler.sample_views(src, poses, K, tposes, seed=a.seed * 1000003 + g[0][0])
            for r, (d, t) in enumerate(ds_g):
                score(d['name'], t, gen[r], d['x'][t])

    with open(os.path.join(a.out, 'metrics.jsonl'), 'w') as fh:
        for rec in records:
            fh.write(json.dumps(rec) + '\n')
    summary = dict(mean_psnr=float(np.mean([r['psnr'] for r in records])) if records else float('nan'),
                   mean_ssim=float(np.mean([r['ssim'] for r in records])) if records else float('nan'),
                   n_views=len(records), prediction='v' if a.distilled or a.consistency else a.prediction,
                   distilled=a.distilled, consistency=a.consistency,
                   cd_steps=cd_steps(a.ckpt) if a.consistency else None, sampler_steps=len(sampler.sched), args=vars(a))
    with open(os.path.join(a.out, 'summary.json'), 'w') as fh:
        json.dump(summary, fh, indent=1)
    print(json.dumps(summary))


if __name__ == '__main__':
    main()
