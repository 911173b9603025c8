"""The four Llama-3-8B decode projections (qkv, o, gate/up, down) on bf16 against fp8 (e4m3) weights, through the kernel entry points:
decode at M = 128 rows (the stream-K GEMM: oa_k_gemm_streamk / oa_k_gemm_streamk_fp8, weight TB/s) and prefill at M = 8192 (the persistent
tile GEMM: oa_k_gemm / oa_k_gemm_fp8, TFLOP/s).  Also the row quantiser (oa_k_quant_rows_e4m3) on each projection's input.

    python tools/w8_fp8_gemm_bench.py [--iters 20] [--ctas 132]

Calls alternate A B A B ...; kernel device times come from torch.profiler (CUDA activity), so the entry points' own allocations, copies and
the test-only partial reduction are not counted.  Prints the card name and power limit beside the times, and one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opsagent_b200 import _lib  # noqa: E402

SHAPES = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}      # (N, K) of Llama-3-8B


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the times are still printed; the card line says why it is missing
        return f"unknown ({e})"


def kernel_ms(prof, must, arm):
    """mean device ms per launch of the kernels whose name contains every string of `must` and the template flag of `arm`"""
    flag = ", true>" if arm == "fp8" else ", false>"
    hits = [e for e in prof.key_averages() if all(m in e.key for m in must) and flag in e.key]
    assert len(hits) == 1, [e.key for e in prof.key_averages()]
    return hits[0].device_time_total / max(1, hits[0].count) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ctas", type=int, default=132)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "decode_m128": {}, "prefill_m8192": {}, "quantiser_ms": {}}

    def q8(x):
        q = torch.empty(x.shape, dtype=torch.uint8, device="cuda"); s = torch.empty(x.shape[0], dtype=torch.float32, device="cuda")
        assert L.oa_k_quant_rows_e4m3(ptr(x), ptr(q), ptr(s), x.shape[0], x.shape[1], None) == 0, _lib.last_error()
        return q, s

    for name, (N, K) in SHAPES.items():
        w = (torch.randn(N, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        qw, sw = q8(w)
        for M, key in ((128, "decode_m128"), (8192, "prefill_m8192")):
            x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
            qx, sx = q8(x)
            if M == 128:
                out = torch.empty(M, N, dtype=torch.float32, device="cuda")
                calls = {"bf16": lambda: L.oa_k_gemm_streamk(ptr(x), ptr(w), M, N, K, 128, a.ctas, ptr(out), None),
                         "fp8": lambda: L.oa_k_gemm_streamk_fp8(ptr(qx), ptr(sx), ptr(qw), ptr(sw), M, N, K, 128, a.ctas, 0, None, ptr(out), None)}
                must = ["gemm_streamk_kernel<128, 1, 0"]
            else:
                out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
                calls = {"bf16": lambda: L.oa_k_gemm(ptr(x), ptr(w), M, N, K, 0, 128, ptr(out), None, None, None, None, None),
                         "fp8": lambda: L.oa_k_gemm_fp8(ptr(qx), ptr(sx), ptr(qw), ptr(sw), M, N, K, 0, 128, ptr(out), None, None, None)}
                must = ["gemm_persistent_kernel<0"]
            for _ in range(2):
                for arm in ("bf16", "fp8"):
                    assert calls[arm]() == 0, _lib.last_error()          # warm-up: module load, smem attributes
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    for arm in ("bf16", "fp8"):
                        calls[arm]()
                    if M == 128:
                        q8(x)
                torch.cuda.synchronize()
            r = {}
            for arm in ("bf16", "fp8"):
                ms = kernel_ms(prof, must, arm)
                wbytes = N * K * (1 if arm == "fp8" else 2) + (4 * N if arm == "fp8" else 0)
                r[arm] = {"ms": round(ms, 4), ("weight_tb_s" if M == 128 else "tflop_s"):
                          round((wbytes / ms / 1e9) if M == 128 else (2.0 * M * N * K / ms / 1e9), 3)}
            r["fp8_over_bf16"] = round(r["fp8"]["ms"] / r["bf16"]["ms"], 3)
            res[key][name] = r
            if M == 128:
                hits = [e for e in prof.key_averages() if "quant_rows_e4m3_kernel" in e.key]
                res["quantiser_ms"][f"{name}_input_128x{K}"] = round(hits[0].device_time_total / max(1, hits[0].count) / 1e3, 4)
    tot = {arm: sum(res["decode_m128"][n][arm]["ms"] for n in SHAPES) for arm in ("bf16", "fp8")}
    res["decode_m128"]["sum_ms"] = {k: round(v, 4) for k, v in tot.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
