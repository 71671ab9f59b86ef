"""Estimates camera poses on SRN with a trained checkpoint (novel_view_synthesis_3d_b200.pose.PoseEstimator), following the
single-view protocol of eval_srn.py: each instance is conditioned on one source view (view 64 by default) at its known pose,
and the pose of every --stride-th other view is estimated from that view's image alone.

    python examples/pose_srn.py cars_test --ckpt checkpoints --prefix ema --side 128 --hypotheses 8 --draws 2 \\
        --iters 200 --stride 25 --max-instances 20 --out pose_eval/
    python examples/pose_srn.py cars_test --ckpt checkpoints_v --prefix ema --side 128 --prediction v --out pose_v/
    python examples/pose_srn.py cars_test --ckpt checkpoints_d6 --prefix ema --side 128 --distilled 6 --out pose_d6/

Writes out/pose.json: one record per (instance, target view) with the rotation error (degrees, geodesic) and the
camera-centre error (scene units) of the best hypothesis, plus the median rotation error, the accuracy at 15 and 30 degrees
and the arguments; prints the summary as the last line of stdout.  Seeds derive from --seed, so equal arguments give equal
files.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import pose as PO
from novel_view_synthesis_3d_b200.srn_data import SRNScenes


def select_targets(n_views: int, source: int, stride: int) -> list:
    """Views 0, stride, 2 stride, ... of an instance with n_views views, without the source."""
    return [v for v in range(0, n_views, max(1, stride)) if v != source]


def pair_errors(R_est, t_est, R_true, t_true) -> dict:
    """Rotation error (degrees) and camera-centre error (distance between the t of two cam-to-world poses) of one pair."""
    return dict(rot_err_deg=float(PO.rotation_error_deg(R_est, R_true)),
                center_err=float(np.linalg.norm(np.asarray(t_est, np.float64) - np.asarray(t_true, np.float64))))


def summarize(records: list) -> dict:
    """Median rotation error and the fraction of pairs within 15 and 30 degrees."""
    e = np.array([r['rot_err_deg'] for r in records], np.float64)
    if e.size == 0:
        return dict(n_pairs=0, median_rot_err_deg=float('nan'), acc_15=float('nan'), acc_30=float('nan'),
                    median_center_err=float('nan'))
    return dict(n_pairs=int(e.size), median_rot_err_deg=float(np.median(e)), acc_15=float(np.mean(e < 15.0)),
                acc_30=float(np.mean(e < 30.0)), median_center_err=float(np.median([r['center_err'] for r in records])))


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('folder')
    ap.add_argument('--ckpt', default='checkpoints')
    ap.add_argument('--prefix', default='model', help="checkpoint prefix: 'ema' reads the weight EMA of train_srn.py")
    ap.add_argument('--side', type=int, default=64)
    ap.add_argument('--prediction', choices=P.sampling.PREDICTIONS, default='eps',
                    help='what the checkpoint predicts: the noise (eps) or v (a model trained with --prediction v)')
    ap.add_argument('--distilled', type=int, default=0, metavar='R',
                    help='a student distilled R times (examples/distill_srn.py): read as v; --prediction is then ignored')
    ap.add_argument('--ray-convention', choices=tuple(P._lib.RAYS), default='v3d130_ij',
                    help='the ray convention the checkpoint was trained with (XUNet(ray_convention=...))')
    ap.add_argument('--source-view', type=int, default=64, help='conditioning view of every instance (pixelNeRF / 3DiM: 64)')
    ap.add_argument('--stride', type=int, default=25, help='estimate the pose of every stride-th view')
    ap.add_argument('--max-instances', type=int, default=-1, help='the first N instances of the sorted list')
    ap.add_argument('--hypotheses', type=int, default=PO.HYPOTHESES)
    ap.add_argument('--draws', type=int, default=PO.DRAWS)
    ap.add_argument('--iters', type=int, default=PO.ITERS)
    ap.add_argument('--lr', type=float, default=PO.LR)
    ap.add_argument('--t-range', type=int, nargs=2, default=list(PO.T_RANGE), metavar=('T_MIN', 'T_MAX'))
    ap.add_argument('--eval-draws', type=int, default=None)
    ap.add_argument('--translate', action='store_true', help='fit the translation too (6 DoF)')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default='pose_eval')
    a = ap.parse_args(argv)
    if a.stride < 1:
        ap.error('--stride must be >= 1')
    return a


def main(argv=None):
    a = parse_args(argv)
    params = P.checkpoint.restore_checkpoint(a.ckpt, prefix=a.prefix)
    if params is None:
        raise FileNotFoundError('Checkpoint does not exist')
    ds = SRNScenes(a.folder, img_sidelength=a.side, max_num_instances=a.max_instances)
    est = PO.PoseEstimator(P.XUNet(ray_convention=a.ray_convention), params, a.side, hypotheses=a.hypotheses, draws=a.draws,
                           prediction='v' if a.distilled else a.prediction, t_range=tuple(a.t_range), lr=a.lr,
                           translate=a.translate, eval_draws=a.eval_draws)
    records = []
    for i in range(len(ds.instances)):
        d = ds.instance_views(i)
        s, n = a.source_view, len(d['x'])
        if s < 0 or s >= n:
            raise SystemExit(f"instance {d['name']} has {n} views; --source-view {s} does not exist")
        for v in select_targets(n, s, a.stride):
            res = est.estimate(d['x'][s], d['R'][s], d['t'][s], d['K'], d['x'][v], iters=a.iters,
                               seed=(a.seed * 1000003 + i) * 1009 + v)
            b = res.best
            rec = dict(instance=d['name'], view=int(v), best=b, score=float(res.score[b]))
            rec.update(pair_errors(res.R[b].cpu().numpy(), res.t[b].cpu().numpy(), d['R'][v], d['t'][v]))
            records.append(rec)
    summary = dict(summarize(records), prediction='v' if a.distilled else a.prediction, distilled=a.distilled, args=vars(a))
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'pose.json'), 'w') as fh:
        json.dump(dict(summary=summary, pairs=records), fh, indent=1)
    print(json.dumps(summary))


if __name__ == '__main__':
    main()
