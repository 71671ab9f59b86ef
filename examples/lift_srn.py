"""Lifts one view of each SRN instance to a radiance grid by score distillation (novel_view_synthesis_3d_b200.lift.FieldLifter)
and scores the grid's renders at the held-out views eval_srn.py scores, against ground truth: each instance is conditioned on
one source view (view 64 by default) at its known pose, the world up and the elevation band of the drawn cameras come from the
instance's own cameras (estimate_up, elevation_range), and after the lift the grid is rendered at the --targets evenly spaced
other views.

    python examples/lift_srn.py cars_test --ckpt checkpoints --prefix ema --side 64 --draws 2 --iters 1000 \\
        --targets 10 --max-instances 20 --out lift_eval/

Writes out/metrics.jsonl (one {instance, view, psnr, ssim} line per scored view, plus the instance's lift diagnostics) and
out/summary.json (mean PSNR, mean SSIM, the number of views and the arguments), prints the summary as the last line of stdout,
and with --save-renders writes each render as out/renders/<instance>_<view>.png.  Seeds derive from --seed, so equal arguments
give equal files.  Whether lifting scores better than sample_views + fit_field on SRN has not been measured.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import lift as LI
from novel_view_synthesis_3d_b200.srn_data import SRNScenes


def select_targets(n_views: int, source: int, count: int) -> list:
    """eval_srn.py's target views: `count` views spaced evenly over the views other than `source`, in increasing order; all of
    them when count is 0 or at least their number."""
    rest = [v for v in range(n_views) if v != source]
    if count <= 0 or count >= len(rest):
        return rest
    return [rest[i] for i in np.linspace(0, len(rest), num=count, endpoint=False, dtype=int)]


def camera_band(R, t):
    """(up, residual, (lo, hi)): the world up of an instance's cameras (estimate_up), its residual, and the elevation band
    of their centres in degrees (elevation_range)."""
    up, res = LI.estimate_up(R)
    return up, res, LI.elevation_range(t, up)


def summarize(records: list) -> dict:
    """Mean PSNR and SSIM over the scored views."""
    if not records:
        return dict(mean_psnr=float('nan'), mean_ssim=float('nan'), n_views=0)
    return dict(mean_psnr=float(np.mean([r['psnr'] for r in records])), mean_ssim=float(np.mean([r['ssim'] for r in records])),
                n_views=len(records))


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('folder')
    ap.add_argument('--ckpt', default='checkpoints')
    ap.add_argument('--prefix', default='model', help="checkpoint prefix: 'ema' reads the weight EMA of train_srn.py")
    ap.add_argument('--side', type=int, default=64)
    ap.add_argument('--prediction', choices=P.sampling.PREDICTIONS, default='eps',
                    help='what the checkpoint predicts: the noise (eps) or v (a model trained with --prediction v)')
    ap.add_argument('--ray-convention', choices=tuple(P._lib.RAYS), default='v3d130_ij',
                    help='the ray convention the checkpoint was trained with (XUNet(ray_convention=...))')
    ap.add_argument('--source-view', type=int, default=64, help='conditioning view of every instance (pixelNeRF / 3DiM: 64)')
    ap.add_argument('--targets', type=int, default=0, help='held-out views per instance, spaced evenly; 0 = all other views')
    ap.add_argument('--max-instances', type=int, default=-1, help='the first N instances of the sorted list')
    ap.add_argument('--draws', type=int, default=LI.DRAWS)
    ap.add_argument('--w', type=float, default=LI.W)
    ap.add_argument('--t-range', type=int, nargs=2, default=list(LI.T_RANGE), metavar=('T_MIN', 'T_MAX'))
    ap.add_argument('--grid', type=int, default=None, help='grid side G (default: --side)')
    ap.add_argument('--iters', type=int, default=LI.ITERS)
    ap.add_argument('--lr', type=float, default=LI.LR)
    ap.add_argument('--tv', type=float, nargs=2, default=list(LI.TV), metavar=('DENSITY', 'COLOUR'))
    ap.add_argument('--sds-weight', type=float, default=1.0)
    ap.add_argument('--recon-weight', type=float, default=1.0)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default='lift_eval')
    ap.add_argument('--save-renders', action='store_true')
    a = ap.parse_args(argv)
    if a.draws < 1:
        ap.error('--draws must be >= 1')
    return a


def main(argv=None):
    a = parse_args(argv)
    params = P.checkpoint.restore_checkpoint(a.ckpt, prefix=a.prefix)
    if params is None:
        raise FileNotFoundError('Checkpoint does not exist')
    ds = SRNScenes(a.folder, img_sidelength=a.side, max_num_instances=a.max_instances)
    lifter = LI.FieldLifter(P.XUNet(ray_convention=a.ray_convention), params, a.side, draws=a.draws, w=a.w,
                            prediction=a.prediction, t_range=tuple(a.t_range), grid=a.grid)
    os.makedirs(a.out, exist_ok=True)
    if a.save_renders:
        os.makedirs(os.path.join(a.out, 'renders'), exist_ok=True)
    records = []
    with open(os.path.join(a.out, 'metrics.jsonl'), 'w') as fh:
        for i in range(len(ds.instances)):
            d = ds.instance_views(i)
            s, n = a.source_view, len(d['x'])
            if s < 0 or s >= n:
                raise SystemExit(f"instance {d['name']} has {n} views; --source-view {s} does not exist")
            targets = select_targets(n, s, a.targets)
            up, up_res, elev = camera_band(d['R'], d['t'])
            res = lifter.lift(d['x'][s], d['R'][s], d['t'][s], d['K'], iters=a.iters, up=up, elevation=elev, lr=a.lr,
                              tv=tuple(a.tv), sds_weight=a.sds_weight, recon_weight=a.recon_weight,
                              seed=a.seed * 1000003 + i)
            if not targets:
                continue
            gen = res.field.render(d['R'][targets], d['t'][targets], d['K'])
            m = P.image_metrics(gen, d['x'][targets])
            for v, psnr, ssim in zip(targets, m['psnr'].tolist(), m['ssim'].tolist()):
                rec = dict(instance=d['name'], view=int(v), psnr=psnr, ssim=ssim, up_residual=up_res,
                           final_sds=float(res.sds[-1]), final_recon=float(res.field.loss[-1]))
                records.append(rec)
                fh.write(json.dumps(rec) + '\n')
            if a.save_renders:
                for v, img in zip(targets, gen.cpu().numpy()):
                    P.sampling.save_view(os.path.join(a.out, 'renders', f"{d['name']}_{v:06d}.png"), img)
    summary = dict(summarize(records), args=vars(a))
    with open(os.path.join(a.out, 'summary.json'), 'w') as fh:
        json.dump(summary, fh, indent=1)
    print(json.dumps(summary))


if __name__ == '__main__':
    main()
