"""Decode and prefill attention on a bf16 against an fp8 (e4m3) paged KV cache, through the kernel entry points
(oa_k_paged_attention / oa_k_paged_attention_fp8), at Llama-3-8B's attention geometry (32 query heads on 8 kv heads, head_dim 128).

    python tools/kv_fp8_attn_bench.py [--batch 128] [--ctx 1664] [--prompts 16] [--prompt-len 1536] [--iters 20]

The two caches hold the same values (the fp8 one quantised from the bf16 one).  Calls alternate A B A B ...; kernel device times come from
torch.profiler (CUDA activity), so the entry points' own allocations and copies are not counted.  Prints the card name and power limit
beside the times, and one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opsagent_b200 import _lib  # noqa: E402

NH, NKV, D = 32, 8, 128


def ptr(t):
    return C.c_void_p(t.data_ptr())


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the times are still printed; the card line says why it is missing
        return f"unknown ({e})"


def caches(num_pages, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    kv = torch.randn(2, num_pages, NKV, 64, D, generator=g).to(torch.bfloat16).cuda()
    k8 = kv[0].float().clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    v8 = kv[1].float().clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    fp8 = torch.stack([k8.reshape(num_pages, NKV, 64 * D), v8.transpose(2, 3).contiguous().reshape(num_pages, NKV, 64 * D)]).contiguous()
    return kv, fp8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--ctx", type=int, default=1664)
    ap.add_argument("--prompts", type=int, default=16)
    ap.add_argument("--prompt-len", type=int, default=1536)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = _lib.load()
    rng = np.random.default_rng(1)

    def setup(n_seqs, ctx, qlens):
        maxp = (max(ctx) + 63) // 64
        num_pages = sum((c + 63) // 64 for c in ctx)
        bt = np.zeros((n_seqs, maxp), np.int32); k = 0
        perm = rng.permutation(num_pages).astype(np.int32)
        for i, c in enumerate(ctx):
            n = (c + 63) // 64; bt[i, :n] = perm[k:k + n]; k += n
        bf, f8 = caches(num_pages)
        q = torch.randn(int(sum(qlens)), NH, D, device="cuda").to(torch.bfloat16)
        out = torch.empty_like(q)
        return dict(maxp=maxp, num_pages=num_pages, bt=bt, bf=bf, f8=f8, q=q, out=out,
                    ctx=np.ascontiguousarray(ctx, np.int32), ql=np.ascontiguousarray(qlens, np.int32), n=n_seqs)

    def call(s, fp8):
        args = (ptr(s["q"]), ptr(s["out"]), ptr(s["f8"] if fp8 else s["bf"]), s["num_pages"], s["bt"].ctypes.data, s["maxp"],
                s["ctx"].ctypes.data, s["ql"].ctypes.data, s["n"], NH, NKV, D, 0)
        rc = L.oa_k_paged_attention_fp8(*args, 1.0, 1.0, None) if fp8 else L.oa_k_paged_attention(*args, None)
        assert rc == 0, _lib.last_error()

    dec_ctx = np.clip(rng.normal(a.ctx, a.ctx * 0.1, a.batch).astype(np.int64), 64, None)
    dec = setup(a.batch, dec_ctx, np.ones(a.batch, np.int32))
    pre = setup(a.prompts, np.full(a.prompts, a.prompt_len), np.full(a.prompts, a.prompt_len))
    for s in (dec, pre):
        for fp8 in (False, True, False, True):
            call(s, fp8)          # warm-up: module load, smem attributes
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(a.iters):
            for s in (dec, pre):
                call(s, False); call(s, True)
        torch.cuda.synchronize()
    times = {}
    for ev in prof.key_averages():
        for kern in ("decode", "prefill"):
            for arg, arm in (("true", "fp8"), ("false", "bf16")):
                if f"{kern}_attention_kernel<{D}, {arg}>" in ev.key:
                    assert f"{kern}_{arm}" not in times, ev.key
                    times[f"{kern}_{arm}"] = ev.device_time_total / max(1, ev.count) / 1e3     # us -> ms per launch
    assert sorted(times) == ["decode_bf16", "decode_fp8", "prefill_bf16", "prefill_fp8"], [e.key for e in prof.key_averages()]
    kv_bytes = float(dec_ctx.sum()) * NKV * D * 2
    res = {"card": card(), "decode_ms": {k: round(v, 4) for k, v in times.items() if k.startswith("decode")},
           "prefill_ms": {k: round(v, 4) for k, v in times.items() if k.startswith("prefill")},
           "decode_kv_gb": {"bf16": round(kv_bytes * 2 / 1e9, 3), "fp8": round(kv_bytes / 1e9, 3)},
           "geometry": {"batch": a.batch, "mean_ctx": float(dec_ctx.mean()), "prompts": a.prompts, "prompt_len": a.prompt_len, "heads": [NH, NKV, D]}}
    if "decode_bf16" in times and "decode_fp8" in times:
        res["decode_fp8_over_bf16"] = round(times["decode_fp8"] / times["decode_bf16"], 3)
        res["decode_tb_s"] = {"bf16": round(kv_bytes * 2 / times["decode_bf16"] / 1e9, 3), "fp8": round(kv_bytes / times["decode_fp8"] / 1e9, 3)}
    if "prefill_bf16" in times and "prefill_fp8" in times:
        res["prefill_fp8_over_bf16"] = round(times["prefill_fp8"] / times["prefill_bf16"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
