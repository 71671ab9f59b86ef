"""Rebuild an EMA of any width from the post-hoc EMA snapshots of a run (train_srn.py / distill_srn.py --posthoc-ema S1 S2),
without training again (Karras et al. 2024, §3; novel_view_synthesis_3d_b200.posthoc).  Writes a params checkpoint in
the model<step> format, which sample_srn.py, eval_srn.py, lift_srn.py and pose_srn.py read with --prefix.

    python examples/posthoc_ema_srn.py --ckpt checkpoints --sigma-rel 0.08 --prefix phema008
    python examples/posthoc_ema_srn.py --ckpt checkpoints --sigma-rel 0.03 --step 50000 --prefix phema003
    python examples/eval_srn.py cars_test --ckpt checkpoints --prefix phema008 ...
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import posthoc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ckpt', required=True, help='directory holding the posthoc<count> snapshots')
    ap.add_argument('--sigma-rel', type=float, required=True, help='relative width of the EMA to rebuild, e.g. 0.08')
    ap.add_argument('--step', type=int, default=None, help='the Adam count to rebuild it at (default: the last snapshot)')
    ap.add_argument('--prefix', required=True, help='prefix of the written checkpoint, e.g. phema008')
    ap.add_argument('--out', default=None, help='directory to write it to (default: --ckpt)')
    a = ap.parse_args()
    if a.prefix == posthoc.SNAPSHOT_PREFIX:
        ap.error(f'--prefix {a.prefix} would be read back as a snapshot')
    if not torch.cuda.is_available():
        raise SystemExit('posthoc_ema_srn.py sums the snapshots on a CUDA device')
    snaps = posthoc.load_snapshots(a.ckpt)
    t = snaps[-1].t if a.step is None else a.step
    print(f'{len(snaps)} snapshots, counts {snaps[0].t}..{snaps[-1].t}, tracked sigma_rel {snaps[-1].sigma_rel}; '
          f'rebuilding sigma_rel {a.sigma_rel:g} (gamma {posthoc.sigma_rel_to_gamma(a.sigma_rel):.4f}) at count {t}')
    tree = posthoc.reconstruct(a.ckpt, a.sigma_rel, t)
    path = P.checkpoint.save_checkpoint(a.out or a.ckpt, tree, step=t, prefix=a.prefix, add_device_axis=True)
    print(f'wrote {path}')


if __name__ == '__main__':
    main()
