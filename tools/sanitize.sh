#!/bin/bash
# compute-sanitizer passes (memcheck + racecheck + synccheck) over the FFT kernels on small parity cases and over the
# fold's kernels (fold_plan_kernel, fold_coherence_kernel, fold_finish_kernel) on small oracle cases (KF).
# usage: tools/sanitize.sh <tag>
TAG=${1:-san}
mkdir -p gpurun_out
KF='(fold_coherence_against_oracle and (1-256 or 8-4096 or 64-7)) or long_call_splits'
K='(fft_c2c_vs_float64 and (1-8-16 or 1-12-5 or 1-14-2 or 1-16-2 or 1-17-2)) or (fft_r2c_inplace_vs_float64 and (16 or 17 or 18)) or chain_vs_oracle or dm_sweep or pipelined or snap1 or golden'
for tool in memcheck racecheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 7 --print-limit 20 \
    python -m pytest tests/test_gpu_parity.py tests/test_golden.py tests/test_gpu_fold_coherence.py -m gpu -q -x \
    --timeout 800 -k "$K or $KF" \
    > gpurun_out/sanitize_${TAG}_$tool.log 2>&1
  echo "$tool rc=$?"; grep -E "ERROR SUMMARY|passed|failed|error" gpurun_out/sanitize_${TAG}_$tool.log | tail -4
done
