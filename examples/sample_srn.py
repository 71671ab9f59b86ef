"""sampling.py look-alike (reference: sampling.py:55-167): restore a Flax-format checkpoint, draw one batch, run the CFG
ancestral sampler, write PNGs (the reference blocks in cv2.imshow, which cannot run headless).

    python examples/sample_srn.py cars_train_val --ckpt checkpoints --steps 256 --out results/
    python examples/sample_srn.py cars_train_val --ckpt checkpoints --prefix ema --steps 256 --out results_ema/
    python examples/sample_srn.py cars_train_val --ckpt checkpoints --method dpmpp_2m --steps 25 --out results_dpm/
    python examples/sample_srn.py cars_train_val --ckpt checkpoints_v --prediction v --method dpmpp_2m --steps 25 --out results_v/
    python examples/sample_srn.py cars_train_val --ckpt checkpoints_d1 --prefix ema --distilled 1 --steps 256 --out results_d1/
    python examples/sample_srn.py cars_train_val --ckpt checkpoints_cd --prefix ema --consistency 2 --out results_cd2/
    python examples/sample_srn.py cars_train_val --ckpt checkpoints --method dpmpp_2m --steps 25 --cache-interval 3 --out results_dc3/
    python examples/posthoc_ema_srn.py --ckpt checkpoints --sigma-rel 0.05 --step 100000 --prefix guide005
    python examples/sample_srn.py cars_train_val --ckpt checkpoints --prefix phema010 --guide-prefix guide005 --w 1 \
        --method dpmpp_2m --steps 25 --out results_ag/
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200.srn_data import SRNScenes

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from distill_srn import cd_steps  # noqa: E402


def add_guide_args(ap) -> None:
    ap.add_argument('--guide-ckpt', default=None, metavar='DIR',
                    help='directory of the autoguidance checkpoint (default: --ckpt)')
    ap.add_argument('--guide-prefix', default=None, metavar='P',
                    help='autoguidance (Karras et al. 2024): guide with this weaker checkpoint of the same model, for '
                         'example a post-hoc EMA at a short sigma_rel and an early step (examples/posthoc_ema_srn.py), in '
                         'place of the pose-dropped branch; --w then weights (1 + w) out - w out_guide')


def load_guide(ap, a):
    """The guide's parameter tree (None without --guide-prefix); argparse errors for a combination that has no guidance."""
    if a.guide_prefix is None:
        if a.guide_ckpt is not None:
            ap.error('--guide-ckpt needs --guide-prefix')
        return None
    if a.distilled or a.consistency:
        ap.error('--guide-prefix guides the classifier-free-guided sampler; --distilled and --consistency sample without '
                 'guidance')
    guide = P.checkpoint.restore_checkpoint(a.guide_ckpt or a.ckpt, prefix=a.guide_prefix)
    if guide is None:
        raise FileNotFoundError(f'Guide checkpoint {a.guide_prefix} does not exist in {a.guide_ckpt or a.ckpt}')
    return guide


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('folder')
    ap.add_argument('--ckpt', default='checkpoints')
    ap.add_argument('--prefix', default='model', help="checkpoint prefix: 'ema' samples the weight EMA of train_srn.py")
    ap.add_argument('--steps', type=int, default=1000)       # the reference runs all 1000 steps, sampling.py:128
    ap.add_argument('--w', type=float, default=3.0)          # sampling.py:133
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
    ap.add_argument('--views', type=int, default=1)
    ap.add_argument('--side', type=int, default=64)
    ap.add_argument('--out', default='results')
    ap.add_argument('--orbit', type=int, default=0,
                    help='3DiM stochastic conditioning: generate this many further views autoregressively (the poses of the '
                         'next pairs drawn from the loader), each denoising step conditioned on a random view of the pool')
    a = ap.parse_args()
    guide = load_guide(ap, a)
    params = P.checkpoint.restore_checkpoint(a.ckpt, prefix=a.prefix)
    if params is None:
        raise FileNotFoundError('Checkpoint does not exist')                                          # sampling.py:111-112
    ds = SRNScenes(a.folder, img_sidelength=a.side, max_observations_per_instance=50)
    batch = next(ds.batches(a.views))
    model = P.XUNet()
    cache = dict(cache_interval=a.cache_interval, cache_level=a.cache_level)
    if a.consistency:
        sampler = P.Sampler(model, params, a.views, a.side, w=None, method='consistency', prediction='v',
                            timesteps=P.consistency_grid(cd_steps(a.ckpt), a.consistency),
                            dynamic_threshold=a.dynamic_threshold, **cache)
    elif a.distilled:
        sampler = P.Sampler(model, params, a.views, a.side, w=None, method='ddim', prediction='v',
                            timesteps=P.distill_grid(a.steps, a.distilled), dynamic_threshold=a.dynamic_threshold, **cache)
    else:
        sampler = P.Sampler(model, params, a.views, a.side, steps=a.steps, w=a.w, method=a.method, eta=a.eta,
                            spacing=a.spacing, dynamic_threshold=a.dynamic_threshold, prediction=a.prediction,
                            guide_params=guide, **cache)
    os.makedirs(a.out, exist_ok=True)
    if a.orbit > 0:
        it = ds.batches(a.views)
        more = [next(it) for _ in range(a.orbit)]
        tp = {'R': np.stack([b['R2'] for b in more], 1), 't': np.stack([b['t2'] for b in more], 1)}
        seq = sampler.sample_views(batch['x'][:, None], {'R': batch['R1'][:, None], 't': batch['t1'][:, None]}, batch['K'], tp)
        for i, views in enumerate(seq.cpu().numpy()):
            for j, img in enumerate(views):
                P.sampling.save_view(os.path.join(a.out, f'object_{i}_view_{j}.png'), img)
        return
    z = sampler.sample(batch)
    for i, img in enumerate(z.cpu().numpy()):
        P.sampling.save_view(os.path.join(a.out, f'view_{i}.png'), img)                               # z/2 + 0.5, sampling.py:153
        P.sampling.save_view(os.path.join(a.out, f'source_{i}.png'), batch['x'][i])


if __name__ == '__main__':
    main()
