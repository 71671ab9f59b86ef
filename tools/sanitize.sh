#!/bin/bash
# compute-sanitizer over the H100 build (run from the repo root where compute-sanitizer can attach): memcheck over smoke() = one
# tiny forward + backward + Adam of the whole network in fp32 (SIMT kernels) and bf16 (wgmma kernels, fused epilogues), and
# memcheck + racecheck + synccheck over the operator-level tensor-core / 3-channel tests at their smallest shapes.
# Logs -> ${1:-sanitizer_logs}/sanitizer_<tool>.log.
# --launch-timeout: the first `import torch` on a fresh machine takes longer than the sanitizer's default 10 s attach window.
set -u
OUT=${1:-sanitizer_logs}
mkdir -p "$OUT"
T=${SANITIZE_TIMEOUT:-200}
SEL='test_conv_tcgen05_fwd_and_dgrad and (case8 or case9) or test_attention_tcgen05_fwd and case0 or test_attention_tcgen05_bwd and case0 or test_fused_qkv or test_three_channel and (case0 or case2 or case8)'
for tool in memcheck racecheck synccheck; do
  log=$OUT/sanitizer_${tool}.log
  : > $log
  if [ $tool = memcheck ]; then
    echo "== compute-sanitizer --tool $tool : smoke()" >> $log
    timeout $T compute-sanitizer --tool $tool --launch-timeout 300 --print-limit 20 python __graft_entry__.py smoke >> $log 2>&1
  fi
  echo "== compute-sanitizer --tool $tool : operator tests" >> $log
  timeout $T compute-sanitizer --tool $tool --launch-timeout 300 --print-limit 20 python -m pytest tests/test_gpu_ops.py -m gpu -q -x -k "$SEL" -p no:cacheprovider >> $log 2>&1
  grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed|smoke OK|timed" $log | sed "s/^/[$tool] /"
done
