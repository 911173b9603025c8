#!/bin/bash
# compute-sanitizer passes over the CUDA path (SURVEY.md 5.2).  Run on a GPU box from the repo root; logs go to gpurun_out/sanitize_*.log.
# Tiny presets only: the sanitizer serialises and instruments every launch (10-100x slower).
export PYTORCH_NO_CUDA_MEMORY_CACHING=1 OA_SKIP_SLOW_PARITY=1
mkdir -p gpurun_out
S="compute-sanitizer --error-exitcode 86 --print-limit 30"
run() {  # name, seconds, tool, command...
  local name=$1 secs=$2 tool=$3; shift 3
  timeout $secs $S --tool $tool --log-file gpurun_out/sanitize_${name}.log "$@" > gpurun_out/sanitize_${name}.out 2>&1
  echo "$name rc=$? $(grep -c 'ERROR SUMMARY' gpurun_out/sanitize_${name}.log) $(grep 'ERROR SUMMARY' gpurun_out/sanitize_${name}.log | tail -1) | $(tail -1 gpurun_out/sanitize_${name}.out)"
}
run memcheck_kernels 420 memcheck python -m pytest tests/test_kernels_gpu.py -x -q
run memcheck_engine 420 memcheck python -m pytest tests/test_engine_gpu.py -x -q -k "greedy_generation or concurrent_requests or grammar_constrained or prefix_cache or preemption or native_front_routes or cluster_splitk and not 1b"
run memcheck_decode_kernels 600 memcheck python -m pytest tests/test_decode_kernels_gpu.py -x -q -k "refuse or kv_write or masked_argmax or (in_kernel_merge and 32-8-64) or (writes_stay and 1b)"
run memcheck_prefill_kernels 600 memcheck python -m pytest tests/test_prefill_kernels_gpu.py -x -q -k "(rmsnorm and 2048) or (embed_gather and 152064)"
run memcheck_tp_kernels 420 memcheck python -m pytest tests/test_tp_kernels_gpu.py -x -q -k "refuse or short_slices"
run memcheck_decode_chain 240 memcheck python -c "
from oracle import oracle as O; from opsagent_b200 import Engine
e = Engine(O.PRESETS['tiny-llama'].engine_json(num_pages=32, max_seq_len=256, max_batch=8, max_step_tokens=128, start_thread=0))
lg, ids = e.debug_decode_logits(6, 150, 3, 24); assert lg.shape == (3, 6, e.info['vocab']) and ids.shape == (3, 6); print('decode chain ok')"
run memcheck_kv_fp8 420 memcheck python -m pytest tests/test_kv_fp8_gpu.py -x -q -k "fp8_paged or kv_write"
run racecheck_kv_fp8 420 racecheck python -m pytest tests/test_kv_fp8_gpu.py -x -q -k "fp8_paged or kv_write"
run memcheck_w8_fp8 420 memcheck python -m pytest tests/test_w8_fp8_gpu.py -x -q -k "quantiser or (gemm_fp8 and not long_k) and (-1-False or -7-False or quantiser)"
run racecheck_w8_fp8 420 racecheck python -m pytest tests/test_w8_fp8_gpu.py -x -q -k "quantiser or (gemm_fp8 and not long_k) and (-1-False or -7-False or quantiser)"
run racecheck_smoke 240 racecheck python -c "import __graft_entry__ as g; g.smoke()"
run synccheck_smoke 240 synccheck python -c "import __graft_entry__ as g; g.smoke()"
run initcheck_smoke 240 initcheck python -c "import __graft_entry__ as g; g.smoke()"
