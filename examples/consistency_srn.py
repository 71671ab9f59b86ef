"""3D consistency score of generated SRN views (3DiM, Watson et al. 2022, section 5): per instance, a radiance grid is fitted to
most of the views examples/eval_srn.py generated and rendered at the poses of the rest, and those renders are scored against
the generated views they stand in for (novel_view_synthesis_3d_b200.consistency).  The same split of the ground-truth images of
the same views is scored too: the ceiling a perfectly consistent set reaches with this grid and fit.

    python examples/eval_srn.py cars_test --ckpt checkpoints --prefix ema --side 128 --mode stochastic --targets 0 \\
        --source-view 64 --out eval_sc/ --save-views
    python examples/consistency_srn.py cars_test --views eval_sc/views --side 128 --source-view 64 --out consistency_sc/

Reads <views>/<instance>_<view>.png (what eval_srn.py --save-views writes) and the poses and intrinsics of those views from the
SRN folder.  The source view is never fitted: the score is about what the model generated.  Views k (in increasing view order)
with k % --every == --every - 1 are held out.  Writes out/consistency.jsonl (one line per instance: the held-out views, their
PSNR / SSIM and means for the generated and the ground-truth views, and the final fit losses) and out/summary.json (mean
PSNR / SSIM of both, the counts and the arguments), and prints the summary as the last line of stdout.  Seeds derive from
--seed, so equal inputs give equal files.
"""
import argparse
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from novel_view_synthesis_3d_b200 import consistency as CS
from novel_view_synthesis_3d_b200.srn_data import SRNScenes, load_rgb


def generated_views(folder: str, name: str, source: int) -> dict:
    """{view index: path} of the saved views of instance `name`, the source view left out."""
    pat = re.compile(re.escape(name) + r'_(\d+)\.png$')
    found = {}
    for f in sorted(os.listdir(folder)):
        m = pat.match(f)
        if m and int(m.group(1)) != source:
            found[int(m.group(1))] = os.path.join(folder, f)
    return dict(sorted(found.items()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('folder', help='the SRN folder the views were generated from (poses and intrinsics)')
    ap.add_argument('--views', required=True, help="eval_srn.py's <out>/views directory")
    ap.add_argument('--side', type=int, default=64)
    ap.add_argument('--source-view', type=int, default=64, help='the conditioning view; it is never fitted')
    ap.add_argument('--max-instances', type=int, default=-1)
    ap.add_argument('--every', type=int, default=8, help='hold out views k with k % every == every - 1')
    ap.add_argument('--grid', type=int, default=None, help='grid side G (default: --side)')
    ap.add_argument('--iters', type=int, default=CS.ITERS)
    ap.add_argument('--rays', type=int, default=CS.RAYS)
    ap.add_argument('--lr', type=float, default=CS.LR)
    ap.add_argument('--background', type=float, default=1.0, help='in [-1, 1]; SRN renders on white (+1)')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default='consistency')
    a = ap.parse_args()
    if a.every < 2:
        ap.error('--every must be >= 2')
    ds = SRNScenes(a.folder, img_sidelength=a.side, max_num_instances=a.max_instances)
    fit = dict(grid=a.grid, iters=a.iters, rays=a.rays, lr=a.lr, background=a.background)
    todo = []
    for i, inst in enumerate(ds.instances):
        found = generated_views(a.views, inst['name'], a.source_view)
        n = len(found)
        if n < a.every or any(v >= len(inst['imgs']) for v in found):
            raise SystemExit(f"instance {inst['name']}: {n} generated views under {a.views} (views {sorted(found)}), need at "
                             f"least --every {a.every} views that exist in the SRN folder")
        todo.append((i, found))
    os.makedirs(a.out, exist_ok=True)
    records = []
    for i, found in todo:
        d = ds.instance_views(i)
        idx = list(found)
        gen = np.stack([load_rgb(p, a.side) for p in found.values()])
        R, t = d['R'][idx], d['t'][idx]
        seed = a.seed * 1000003 + i
        s = CS.consistency_score(gen, R, t, d['K'], every=a.every, seed=seed, **fit)
        g = CS.consistency_score(d['x'][idx], R, t, d['K'], every=a.every, seed=seed, **fit)
        records.append(dict(instance=d['name'], views=idx, held_out=[idx[k] for k in s['held_out']], psnr=s['psnr'],
                            ssim=s['ssim'], mean_psnr=s['mean_psnr'], mean_ssim=s['mean_ssim'], fit_loss=s['fit_loss'],
                            gt_psnr=g['psnr'], gt_ssim=g['ssim'], gt_mean_psnr=g['mean_psnr'], gt_mean_ssim=g['mean_ssim'],
                            gt_fit_loss=g['fit_loss']))
    with open(os.path.join(a.out, 'consistency.jsonl'), 'w') as fh:
        for rec in records:
            fh.write(json.dumps(rec) + '\n')

    def mean(key):
        return float(np.mean([r[key] for r in records])) if records else float('nan')
    summary = dict(mean_psnr=mean('mean_psnr'), mean_ssim=mean('mean_ssim'), gt_mean_psnr=mean('gt_mean_psnr'),
                   gt_mean_ssim=mean('gt_mean_ssim'), n_instances=len(records),
                   n_held_out=sum(len(r['held_out']) for r in records), args=vars(a))
    with open(os.path.join(a.out, 'summary.json'), 'w') as fh:
        json.dump(summary, fh, indent=1)
    print(json.dumps(summary))


if __name__ == '__main__':
    main()
