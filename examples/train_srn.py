"""train.py look-alike on the CUDA path (reference: train.py:78-176).  Differences from the reference script: imports,
a sharded batch under torchrun, device-side forward diffusion, and Flax-format checkpoints every `save_every` steps: the
params (model<step>), the weight EMA with --ema-decay (ema<step>, a params tree like model<step>), and the whole training
state (state<step>: params, Adam moments and count, EMA, cond_mask streams) that --resume continues from.

    python examples/train_srn.py cars_train_val --batch 8 --side 64 --steps 1000 --ema-decay 0.9999
    python examples/train_srn.py cars_train_val --batch 8 --side 64 --steps 2000 --ema-decay 0.9999 --resume
    python examples/train_srn.py cars_train_val --batch 8 --side 64 --max-grad-norm 1 --warmup-steps 5000 --ema-decay 0.9999
    python examples/train_srn.py cars_train_val --batch 8 --side 64 --posthoc-ema 0.05 0.10 --snapshot-every 1000
    python examples/train_srn.py cars_train_val --batch 4 --side 128 --grad-accum-steps 8     # 32 samples per update
    python examples/train_srn.py cars_train_val --batch 8 --side 64 --loss mse --min-snr-gamma 5
    python examples/train_srn.py cars_train_val --batch 8 --side 64 --loss mse --prediction v --device-data
    python examples/train_srn.py cars_train_val --batch 8 --side 64 --device-data --data-cache cars64.cache
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_srn.py cars_train_val
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import dist as xdist
from novel_view_synthesis_3d_b200.srn_data import SRNScenes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('folder')
    ap.add_argument('--batch', type=int, default=2)          # Trainer(train_batch_size=2), train.py:84
    ap.add_argument('--side', type=int, default=64)          # img_sidelength=64, :88
    ap.add_argument('--lr', type=float, default=1e-4)        # train_lr, :85
    ap.add_argument('--steps', type=int, default=100000)     # train_num_steps, :86
    ap.add_argument('--save-every', type=int, default=1000)  # :87
    ap.add_argument('--dtype', default='bf16')
    ap.add_argument('--ema-decay', type=float, default=None,
                    help='keep an exponential moving average of the weights (e.g. 0.9999) and save it as ema<step>')
    ap.add_argument('--posthoc-ema', type=float, nargs=2, default=None, metavar=('S1', 'S2'),
                    help='keep two power-function averages of the weights of these relative widths (e.g. 0.05 0.10) and '
                         'save snapshots of both, from which posthoc_ema_srn.py rebuilds an EMA of any width after training')
    ap.add_argument('--snapshot-every', type=int, default=1000,
                    help='with --posthoc-ema: write a snapshot of both averages every this many updates (posthoc<count>)')
    ap.add_argument('--max-grad-norm', type=float, default=None,
                    help='clip the gradient to this global L2 norm (e.g. 1) and skip updates whose norm is not finite')
    ap.add_argument('--warmup-steps', type=int, default=0,
                    help='warm the learning rate up linearly from 0 over this many steps (e.g. 5000)')
    ap.add_argument('--grad-accum-steps', type=int, default=1,
                    help='accumulate the gradient over this many micro-batches of --batch samples per update')
    ap.add_argument('--loss', choices=('frobenius', 'mse'), default='frobenius',
                    help="training loss: the reference's ||eps_hat - noise||_F, or the mean squared error of DDPM / 3DiM")
    ap.add_argument('--min-snr-gamma', type=float, default=None,
                    help='with --loss mse: weight each sample by min(SNR_t, G) / SNR_t, or min(SNR_t, G) / (SNR_t + 1) with '
                         '--prediction v (min-SNR-gamma, e.g. 5)')
    ap.add_argument('--prediction', choices=P.sampling.PREDICTIONS, default='eps',
                    help='what the network learns to predict: the noise (eps) or v = sqrt(abar) eps - sqrt(1 - abar) x0 '
                         '(needs --loss mse; sample the checkpoints with --prediction v)')
    ap.add_argument('--device-data', action='store_true',
                    help='decode every view once into GPU memory and draw, gather and noise each batch inside the step; '
                         'the ranks then split one global batch per update instead of each reading its own stream')
    ap.add_argument('--data-cache', default=None, help='with --device-data: directory of the decoded views, reused by later runs')
    ap.add_argument('--data-seed', type=int, default=0, help='with --device-data: seed of the data order')
    ap.add_argument('--resume', action='store_true', help='continue from the latest state<step> checkpoint')
    ap.add_argument('--ckpt', default='checkpoints')
    a = ap.parse_args()
    if a.min_snr_gamma is not None and a.loss != 'mse':
        ap.error('--min-snr-gamma needs --loss mse')
    if a.prediction == 'v' and a.loss != 'mse':
        ap.error('--prediction v needs --loss mse')
    if a.posthoc_ema is not None and a.ema_decay is not None:
        ap.error('--posthoc-ema and --ema-decay are exclusive')
    if a.snapshot_every < 1:
        ap.error('--snapshot-every must be >= 1')
    local = xdist.init_from_env('nccl')
    rank, world = xdist.rank(), xdist.world_size()
    model = P.XUNet(dtype=a.dtype)
    state = P.create_train_state(0, 1, a.lr, a.batch, a.side, model=model, ema_decay=a.ema_decay,
                                 max_grad_norm=a.max_grad_norm, warmup_steps=a.warmup_steps, loss=a.loss,
                                 prediction=a.prediction, posthoc_ema=a.posthoc_ema)
    if a.resume and P.checkpoint.restore_train_state(a.ckpt, state) is not None and rank == 0:
        print(f'resumed from step {state.step}')
    if a.device_data:
        # the data order follows (--data-seed, update count), so --resume continues it exactly
        store = P.DeviceScenes(a.folder, a.side, max_observations_per_instance=50, cache=a.data_cache)
        step = P.TrainStep(state, grad_accum_steps=a.grad_accum_steps, data=store, data_seed=a.data_seed,
                           min_snr_gamma=a.min_snr_gamma)
        for it in range(state.step, a.steps):
            loss = step()
            report(a, state, step, it, loss, rank)
        finish(state, rank)
        return
    ds = SRNScenes(a.folder, img_sidelength=a.side, max_observations_per_instance=50, seed=rank)      # train.py:99-104
    step = P.TrainStep(state, grad_accum_steps=a.grad_accum_steps)
    fd = P.ForwardDiffusion(step.eng, min_snr_gamma=a.min_snr_gamma, prediction=a.prediction)   # 'noise' holds v for v
    dev_keys = ('z', 'logsnr', 'noise', 'cond_mask') + (('loss_weight',) if fd.loss_weight is not None else ())
    stream = ds.batches(a.batch)
    k = a.grad_accum_steps
    for it in range(state.step, a.steps):
        micro = []
        for j in range(k):                                     # one update = k micro-batches of --batch samples
            b = next(stream)
            fd.sample(b['target'], seed=(it * k + j) * world + rank)     # z, noise, logsnr, cond_mask on the GPU
            dev = step.eng.inp
            m = {key: b[key] for key in ('x', 'R1', 't1', 'R2', 't2', 'K')}
            m.update({key: dev[key] if k == 1 else dev[key].clone() for key in dev_keys})
            micro.append(m)
        if k == 1:
            batch = micro[0]
        else:
            batch = {key: torch.cat([m[key] for m in micro]) if isinstance(micro[0][key], torch.Tensor)
                     else np.concatenate([m[key] for m in micro]) for key in micro[0]}
        noise, cond_mask, weight = batch.pop('noise'), batch.pop('cond_mask'), batch.pop('loss_weight', None)
        loss = step(batch, noise, cond_mask=cond_mask, loss_weight=weight)
        report(a, state, step, it, loss, rank)
    finish(state, rank)


def report(a, state, step, it, loss, rank):
    """The loss every 50 updates, the checkpoints every --save-every and, with --posthoc-ema, a snapshot of both averages
    every --snapshot-every updates."""
    if rank == 0 and it % 50 == 0:
        norm = '' if step.grad_norm is None else f'  grad norm {float(step.grad_norm):.4f}'
        print(f'{it}: {float(loss):.4f}{norm}')                                                    # train.py:157
    if it % a.save_every == 0:
        if rank == 0:
            P.checkpoint.save_checkpoint(a.ckpt, state.params, step=it, prefix='model', add_device_axis=True)
            if state.ema_params is not None:
                P.checkpoint.save_checkpoint(a.ckpt, state.ema_params, step=it, prefix='ema', add_device_axis=True)
        P.checkpoint.save_train_state(a.ckpt, state, step=state.step)    # collective: every rank calls it
    if state.posthoc is not None and state.opt_state.count % a.snapshot_every == 0:
        P.posthoc.save_snapshot(a.ckpt, state)                           # rank 0 writes


def finish(state, rank):
    if rank == 0:
        if state.clip is not None:
            print(f'skipped steps (non-finite gradient norm): {state.skipped_steps}')
        print('training completed')


if __name__ == '__main__':
    main()
