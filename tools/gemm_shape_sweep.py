"""Kernel-level sweep of the tile GEMM's N-tile choice for decode-sized batches that fall off the stream-K path (128 < M <= 256):
Qwen2.5-32B TP=4 at B=256 runs its projections on gemm_wgmma_kernel (one CTA per 128 x BN tile), where a few hundred CTAs on 132 SMs
lose up to half a wave.  For each per-rank shape and BN in {32, 64, 128, 256}: CUDA-event time over rotating weight copies (so that
weights come from HBM, as in a real step), against the weight-streaming floor.   python tools/gemm_shape_sweep.py [M]"""
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opsagent_b200 import _lib  # noqa: E402

L = _lib.load()
M = int(sys.argv[1]) if len(sys.argv) > 1 else 256
peak = 6576.1
try:
    peak = float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass
# (name, N, K, epilogue) per rank of Qwen2.5-32B TP=4 and Llama-3-70B TP=8
SHAPES = [("qwen32b/tp4 qkv", 1792, 5120, 0), ("qwen32b/tp4 o", 5120, 1280, 0), ("qwen32b/tp4 gate_up", 13824, 5120, 2), ("qwen32b/tp4 down", 5120, 6912, 0),
          ("llama70b/tp8 qkv", 1280, 8192, 0), ("llama70b/tp8 o", 8192, 1024, 0), ("llama70b/tp8 gate_up", 7168, 8192, 2), ("llama70b/tp8 down", 8192, 3584, 0)]
dev = torch.device("cuda")
stream = torch.cuda.current_stream().cuda_stream
for name, N, K, epi in SHAPES:
    copies = max(2, int(400e6 // (N * K * 2)) + 1)            # > 3 x L2 worth of weights in rotation
    Ws = [torch.randn(N, K, device=dev, dtype=torch.bfloat16) * 0.02 for _ in range(copies)]
    A = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
    out = torch.empty(M, N if epi != 2 else N // 2, device=dev, dtype=torch.bfloat16)
    row = {"shape": name, "M": M, "N": N, "K": K, "floor_us": round(N * K * 2 / peak / 1e3, 1)}
    for bn in (32, 64, 128, 256):
        def run(i):
            rc = L.oa_k_gemm(A.data_ptr(), Ws[i % copies].data_ptr(), M, N, K, epi, bn, out.data_ptr(), None, None, None, None, stream)
            assert rc == 0, _lib.last_error()
        for i in range(3):
            run(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for i in range(n):
            run(i)
        e1.record(); torch.cuda.synchronize()
        tiles = ((N + bn - 1) // bn) * ((M + 127) // 128)
        row[f"bn{bn}_us"] = round(e0.elapsed_time(e1) * 1e3 / n, 1)
        row[f"bn{bn}_ctas"] = tiles
    print(json.dumps(row), flush=True)
    del Ws
