"""Child process of tests/test_forward_chain_gpu.py — run as `python tests/chain_worker.py CASE OUT.npz REPEAT`.

Runs one case of the forward's launch chain on one GPU and writes what it computed to OUT.npz:
- the decode steps of bench_decode's workload (oa_debug_decode_logits): ids [steps, batch], one SHA-256 per logits row, and the full fp32
  logits of the first step and of the last one, which is a mixed step (the batch's decode rows + one new sequence's prefill chunk);
- a fresh 2048-token prefill (the tile path: persistent GEMM, prefill attention, KV writer): one SHA-256 per logits row, the arg-max and
  the maximum of every row.
With REPEAT > 1 the whole case runs that many times in this process; run k's arrays are stored under the prefix "r{k}_".

OA_PDL is read once per process, which is why this is a separate process: the test runs it once as is (programmatic dependent launch on
every kernel) and once with OA_PDL=0 (fully serialised launches) and requires the two to agree bit for bit.  Prints CHAIN_OK on success."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# one rank of Qwen2.5-32B at TP=4 and of Llama-3-70B at TP=8: the per-rank column-parallel shards (heads, ffn, vocab) at full hidden width
QWEN_TP4_RANK = dict(model="qwen-tp4-rank", hidden=5120, n_layers=2, n_heads=10, n_kv_heads=2, head_dim=128, ffn=6912, vocab=38016,
                     qkv_bias=1, rope_theta=1e6, rms_eps=1e-6, norm_random=1, template="chatml")
LLAMA70_TP8_RANK = dict(model="llama70-tp8-rank", hidden=8192, n_layers=2, n_heads=8, n_kv_heads=1, head_dim=128, ffn=3584, vocab=16032,
                        norm_random=1)

# name -> (engine config, batch, ctx_len); every case runs 4 decode steps, the last one mixed with a 64-token prefill chunk
CASES = {
    # what bench.py times (ctx_len = its default ctx0): stream-K projections + consumers, decode plan with cut items and in-kernel merges
    "bench": (dict(model="llama-3-8b"), 128, 1629),
    # opt-in finishing paths: fused stream-K finishers, cluster split-K, L2 prefetch of the weights ahead of the dependency wait
    "opt_in_paths": (dict(model="llama-3-8b", sk_fuse_epi=7, sk_clusterk=7, sk_clusterk_min_fill=0, sk_l2_prefetch_kb=256), 8, 300),
    # activation quantiser -> W8A8 GEMM (the scale wait), fp8 KV cache
    "fp8": (dict(model="llama-3-8b", weight_dtype="fp8_e4m3", kv_cache_dtype="fp8_e4m3"), 64, 1000),
    # tied head, head_dim 64, llama3 RoPE scaling
    "llama_1b": (dict(model="llama-3.2-1b"), 16, 700),
    # 256 decode rows: the tile path (T > 128); then the opt-in two-row-tile stream-K GEMM on the same batch
    "qwen_tp4_rank": (QWEN_TP4_RANK, 256, 2048),
    "qwen_tp4_rank_sk256": (dict(QWEN_TP4_RANK, sk_max_rows=256), 256, 2048),
    # the decode plan of the 70B TP=8 benchmark config: every (sequence, kv head) item cut into several pieces
    "llama70_tp8_rank": (LLAMA70_TP8_RANK, 64, 16896),
}
STEPS, MIXED_ROWS, PREFILL_TOKENS = 4, 64, 2048


def digests(logits: np.ndarray) -> np.ndarray:
    """one SHA-256 per row of the last axis"""
    rows = np.ascontiguousarray(logits).reshape(-1, logits.shape[-1])
    return np.array([hashlib.sha256(r.tobytes()).digest() for r in rows], dtype="S32").reshape(logits.shape[:-1])


def run_case(name: str) -> dict:
    from opsagent_b200 import Engine
    cfg, batch, ctx_len = CASES[name]
    max_seq_len = (ctx_len + STEPS + 1 + 63) // 64 * 64
    pages = batch * (max_seq_len // 64) + (MIXED_ROWS + 63) // 64 + PREFILL_TOKENS // 64 + 1
    eng = Engine(dict(cfg, seed=1234, num_pages=pages, max_seq_len=max(max_seq_len, PREFILL_TOKENS + 64), max_batch=batch + 1,
                      max_step_tokens=8192, prefix_cache=0, start_thread=0))
    logits, ids = eng.debug_decode_logits(batch, ctx_len, STEPS, MIXED_ROWS)
    vocab = eng.info["vocab"]
    toks = ((np.arange(PREFILL_TOKENS, dtype=np.int64) * 2654435761 + 12345) % vocab).astype(np.int32)
    pre = eng.debug_prefill_logits(toks)
    eng.close()
    return {"ids": ids, "digests": digests(logits), "first_step": logits[0].copy(), "mixed_step": logits[-1].copy(),
            "prefill_digests": digests(pre), "prefill_argmax": pre.argmax(axis=1).astype(np.int32), "prefill_max": pre.max(axis=1)}


def main():
    name, out, repeat = sys.argv[1], sys.argv[2], int(sys.argv[3])
    runs = {}
    for k in range(repeat):
        res = run_case(name)
        if not (np.isfinite(res["first_step"]).all() and np.isfinite(res["mixed_step"]).all() and np.isfinite(res["prefill_max"]).all()):
            print(f"{name}: non-finite logits in run {k}", flush=True)
            sys.exit(2)
        runs.update({f"r{k}_{key}": v for key, v in res.items()})
    np.savez(out, **runs)
    print("CHAIN_OK", flush=True)


if __name__ == "__main__":
    main()
