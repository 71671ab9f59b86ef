"""One round of progressive distillation (Salimans & Ho 2022) on SRN: a v-prediction student learns to take one DDIM step
for two of its teacher's, from views held in GPU memory, with every draw, teacher forward and target inside the captured
training step (novel_view_synthesis_3d_b200.distill).  Writes model<step> / ema<step> / state<step> checkpoints like
train_srn.py; --resume continues a round from its latest state<step>.

Round 1 distils the original guided model (its model or ema checkpoint, --w 3, --teacher-prediction eps) from the 2N-step
DDIM grid of Schedule(--teacher-steps) into an N-step student that needs no guidance.  Round r > 1 distils the student of
round r - 1 (v, unguided).  Sample a round-r student with `sample_srn.py --steps <teacher-steps> --distilled r`.

    python examples/distill_srn.py cars_train_val --teacher-ckpt checkpoints --teacher-prefix ema --round 1 --w 3 \\
        --batch 8 --side 64 --steps 20000 --ema-decay 0.9999 --ckpt checkpoints_d1
    python examples/distill_srn.py cars_train_val --teacher-ckpt checkpoints_d1 --teacher-prefix ema --round 2 \\
        --batch 8 --side 64 --steps 20000 --ema-decay 0.9999 --ckpt checkpoints_d2

--consistency N runs consistency distillation (Song et al. 2023, Consistency Models; distill.ConsistencyTeacher) instead of
a progressive round: the original guided model (--w, --teacher-prediction) on the N-step DDIM grid distill_grid(N, 0)
teaches, in one run, a v student that samples in 1-4 steps without guidance.  Sample it with `sample_srn.py --consistency K`
(or `eval_srn.py --consistency K`), which read N from the run's state<step> checkpoint.

    python examples/distill_srn.py cars_train_val --teacher-ckpt checkpoints --teacher-prefix ema --consistency 256 --w 3 \\
        --batch 8 --side 64 --steps 20000 --ema-decay 0.9999 --ckpt checkpoints_cd
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import novel_view_synthesis_3d_b200 as P
from novel_view_synthesis_3d_b200 import dist as xdist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_srn import finish, report  # noqa: E402


def cd_steps(ckpt: str) -> int:
    """N of a consistency-distilled run: the 'cd_steps' of the distillation record in the latest state<step> checkpoint of
    the directory `ckpt` (or in the state file `ckpt`)."""
    path = ckpt if os.path.isfile(ckpt) else P.checkpoint.latest_checkpoint(ckpt, 'state')
    if path is None:
        raise FileNotFoundError(f'no state<step> checkpoint in {ckpt}: the distillation record of a consistency student is '
                                f'read from it')
    with open(path, 'rb') as fh:
        rec = P.checkpoint.msgpack_restore(fh.read()).get('distill') or {}
    if 'cd_steps' not in rec:
        raise ValueError(f'{path} does not hold a consistency-distilled model (distillation record {rec or None})')
    return int(rec['cd_steps'])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('folder')
    ap.add_argument('--teacher-ckpt', required=True, help='directory (or file) of the teacher: the original model or the '
                                                           'student of the previous round')
    ap.add_argument('--teacher-prefix', default='ema', help="the teacher checkpoint's prefix: 'model' or 'ema'")
    ap.add_argument('--teacher-steps', type=int, default=256, help='DDIM steps of the original teacher (round 1 halves them)')
    ap.add_argument('--round', type=int, default=1, help='the round this run trains: 1 distils the original model')
    ap.add_argument('--consistency', type=int, default=0, metavar='N',
                    help='consistency distillation on the N-step teacher grid instead of a progressive round (--teacher-steps '
                         'and --round are then ignored)')
    ap.add_argument('--w', type=float, default=3.0, help='round 1: the guidance weight the student learns to reproduce')
    ap.add_argument('--teacher-prediction', choices=P.sampling.PREDICTIONS, default='eps',
                    help='round 1: what the original model predicts (later teachers are v students)')
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--side', type=int, default=64)
    ap.add_argument('--lr', type=float, default=1e-4)
    ap.add_argument('--steps', type=int, default=20000)
    ap.add_argument('--save-every', type=int, default=1000)
    ap.add_argument('--dtype', default='bf16')
    ap.add_argument('--ema-decay', type=float, default=None)
    ap.add_argument('--posthoc-ema', type=float, nargs=2, default=None, metavar=('S1', 'S2'),
                    help="keep two power-function averages of the student's weights (see train_srn.py --posthoc-ema)")
    ap.add_argument('--snapshot-every', type=int, default=1000)
    ap.add_argument('--max-grad-norm', type=float, default=None)
    ap.add_argument('--warmup-steps', type=int, default=0)
    ap.add_argument('--grad-accum-steps', type=int, default=1)
    ap.add_argument('--data-cache', default=None, help='directory of the decoded views, reused by later runs')
    ap.add_argument('--data-seed', type=int, default=0)
    ap.add_argument('--resume', action='store_true', help='continue from the latest state<step> checkpoint')
    ap.add_argument('--ckpt', default='checkpoints_distill')
    a = ap.parse_args()
    if a.round < 1:
        ap.error('--round must be >= 1')
    if a.consistency < 0 or a.consistency == 1:
        ap.error('--consistency N needs N >= 2')
    if a.posthoc_ema is not None and a.ema_decay is not None:
        ap.error('--posthoc-ema and --ema-decay are exclusive')
    if a.snapshot_every < 1:
        ap.error('--snapshot-every must be >= 1')
    xdist.init_from_env('nccl')
    rank = xdist.rank()
    params = P.checkpoint.restore_checkpoint(a.teacher_ckpt, prefix=a.teacher_prefix)
    if params is None:
        raise FileNotFoundError(f'no {a.teacher_prefix}<step> checkpoint in {a.teacher_ckpt}')
    model = P.XUNet(dtype=a.dtype)
    first = a.round == 1
    if a.consistency:
        teacher = P.ConsistencyTeacher(model, params, a.consistency, batch_size=a.batch, img_sidelength=a.side, w=a.w,
                                       prediction=a.teacher_prediction)
    else:
        teacher = P.Teacher(model, params, a.teacher_steps, batch_size=a.batch, img_sidelength=a.side,
                            w=a.w if first else None, prediction=a.teacher_prediction if first else 'v', rounds=a.round - 1)
    del params
    state = P.create_distill_state(teacher, a.lr, ema_decay=a.ema_decay, max_grad_norm=a.max_grad_norm,
                                   warmup_steps=a.warmup_steps, posthoc_ema=a.posthoc_ema)
    if rank == 0 and a.consistency:
        print(f'consistency distillation: teacher DDIM on {len(teacher.grid)} timesteps (w = {a.w:g})')
    elif rank == 0:
        print(f'round {a.round}: teacher DDIM on {len(teacher.grid)} timesteps '
              f'({"w = %g" % a.w if first else "unguided"}), student on {len(teacher.student_grid)}')
    if a.resume and P.checkpoint.restore_train_state(a.ckpt, state) is not None and rank == 0:
        print(f'resumed from step {state.step}')
    store = P.DeviceScenes(a.folder, a.side, max_observations_per_instance=50, cache=a.data_cache)
    step = P.TrainStep(state, grad_accum_steps=a.grad_accum_steps, data=store, data_seed=a.data_seed, teacher=teacher)
    for it in range(state.step, a.steps):
        loss = step()
        report(a, state, step, it, loss, rank)
    finish(state, rank)


if __name__ == '__main__':
    main()
