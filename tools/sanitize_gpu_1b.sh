#!/bin/bash
# memcheck with real multi-CTA tile splits: llama-3.2-1b puts stream-K pieces of one tile on several of the 132 SMs, so the per-tile flags and the
# CTA-ordered sums of the default (fused SwiGLU) path run under the sanitizer's perturbed timing; variants must stay bit-identical.
export PYTORCH_NO_CUDA_MEMORY_CACHING=1 OA_SKIP_SLOW_PARITY=1
mkdir -p gpurun_out
timeout 560 compute-sanitizer --error-exitcode 86 --print-limit 30 --tool memcheck --log-file gpurun_out/sanitize_memcheck_1b.log \
  python -m pytest tests/test_engine_gpu.py -q -x -k "fused_decode_epilogues and 1b" > gpurun_out/sanitize_memcheck_1b.out 2>&1
echo "memcheck_1b rc=$? | $(grep SUMMARY gpurun_out/sanitize_memcheck_1b.log | tail -1) | $(tail -1 gpurun_out/sanitize_memcheck_1b.out)"
