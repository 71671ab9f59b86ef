#!/bin/bash
# BASELINE.json configs[4]: per-GPU batch sweep 1-64 at 64x64 and 128x128 (small model) and 1-8 for the full 3DiM model at 128x128.
# usage (on a GPU box, repo root): tools/batch_sweep.sh [N_GPUS] > sweep.jsonl     (one bench JSON line per config)
N=${1:-1}
run() {
  if [ "$N" = "1" ]; then python bench.py "$@"
  else python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29731 bench.py --gpus $N "$@"; fi
}
COMMON="--steps 10 --warmup 3 --no-full128 --skip-cpu-baseline --sampler-steps 0"
# SWEEP_SHORT=1: 64x64 and the full model only (GPU-minute budget)
WL="small64 small128"; [ -n "${SWEEP_SHORT:-}" ] && WL="small64"
for W in $WL; do
  for B in 1 2 4 8 16 32 64; do run --workload $W --batch $B $COMMON 2>/dev/null; done
done
for B in 1 2 4 8; do run --workload full128 --batch $B --steps 6 --warmup 3 --skip-cpu-baseline --sampler-steps 0 2>/dev/null; done
