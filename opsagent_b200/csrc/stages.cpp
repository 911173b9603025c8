// stages.cpp — see stages.hpp.
#include "stages.hpp"

#include <cmath>

namespace oa {

void cuda_check(cudaError_t e, const char* what) {
    if (e != cudaSuccess) throw CudaError(e, std::string(what) + ": " + cudaGetErrorString(e));
}

static void mark_if(const Mark& mark, int id) { if (mark) mark(id); }

const RowParallelOp kOProj = {
    6, "o gemm + residual (cluster split-K)", "o gemm + residual (stream-K)", "o gemm (stream-K)", "rmsnorm2", "resid+rmsnorm2", "o partial -> multicast buffer",
    "in-switch allreduce+resid+rmsnorm2", "o partial -> symmetric buffer (bf16)", "o partial -> symmetric buffer", "allreduce+resid+rmsnorm2"};
const RowParallelOp kDownProj = {
    10, "down gemm + residual (cluster split-K)", "down gemm + residual (stream-K)", "down gemm (stream-K)", "rmsnorm1", "resid+rmsnorm1", "down partial -> multicast buffer",
    "in-switch allreduce+resid+rmsnorm1", "down partial -> symmetric buffer (bf16)", "down partial -> symmetric buffer", "allreduce+resid+rmsnorm1"};

void finish_row_parallel(const SkGemm& g, void* x, const void* gain, void* xn, float eps, const RowParallelOp& op, cudaStream_t s, const Mark& mark) {
    if (g.path == 0) {
        cuda_check(launch_gemm_streamk(g.tmA, g.tmB, g.M, g.N, g.K, g.sk, s, g.w8), op.gemm); mark_if(mark, op.mark);
        cuda_check(launch_sk_resid_rmsnorm(g.sk, x, gain, xn, g.M, g.N, eps, s), op.resid);
    } else {
        if (g.path >= 2) cuda_check(launch_gemm_clusterk_resid(g.tmA, g.tmB, g.M, g.N, g.K, g.path, x, g.N, s), op.clusterk);
        else cuda_check(launch_gemm_streamk_resid(g.tmA, g.tmB, g.M, g.N, g.K, g.sk, x, g.N, g.tile_flags, s, g.w8), op.fused);
        mark_if(mark, op.mark);
        cuda_check(launch_rmsnorm_wide(x, gain, xn, g.M, g.N, eps, s), op.norm);
    }
    mark_if(mark, 7);
}

void tp_row_parallel_partial(const SkGemm& g, bool bf16, void* partial, const TpComm::Signal& sg, const RowParallelOp& op, cudaStream_t s,
                             const Mark& mark) {
    cuda_check(launch_gemm_streamk(g.tmA, g.tmB, g.M, g.N, g.K, g.sk, s, g.w8), op.gemm); mark_if(mark, op.mark);
    if (bf16) cuda_check(launch_sk_reduce_bf16(g.sk, partial, g.M, g.N, s, &sg), op.bf16_part);
    else cuda_check(launch_sk_reduce_f32(g.sk, static_cast<float*>(partial), g.M, g.N, s, &sg), op.f32_part);
}

void tp_row_parallel_finish(void* const* peer_partials, int t, bool bf16, void* x, const void* gain, void* xn, int M, int N, float eps,
                            const TpComm::Signal& sg, const RowParallelOp& op, cudaStream_t s, const Mark& mark) {
    if (bf16) cuda_check(launch_ar_resid_rmsnorm_bf16in(peer_partials, t, x, gain, xn, M, N, eps, s, &sg), op.ar);
    else cuda_check(launch_ar_resid_rmsnorm(peer_partials, t, x, gain, xn, M, N, eps, s, &sg), op.ar);
    mark_if(mark, 7);
}

void qkv_rope(const SkGemm& g, const void* bias, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin,
              void* q_out, const KvLayout& kv, int layer, int nh, cudaStream_t s, const Mark& mark) {
    if (g.path == 0) {
        cuda_check(launch_gemm_streamk(g.tmA, g.tmB, g.M, g.N, g.K, g.sk, s, g.w8), "qkv gemm (stream-K)"); mark_if(mark, 2);
        cuda_check(launch_sk_rope_kv_write(g.sk, bias, positions, slots, rope_cos, rope_sin, q_out, kv, layer, g.M, nh, s), "rope (stream-K)"); mark_if(mark, 3);
        return;
    }
    const SkRopeArgs rope = make_sk_rope_args(bias, positions, slots, rope_cos, rope_sin, q_out, kv, layer, nh);
    if (g.path >= 2) cuda_check(launch_gemm_clusterk_rope(g.tmA, g.tmB, g.M, g.N, g.K, g.path, rope, s), "qkv gemm + RoPE + KV write (cluster split-K)");
    else cuda_check(launch_gemm_streamk_rope(g.tmA, g.tmB, g.M, g.N, g.K, g.sk, rope, g.tile_flags, s, g.w8), "qkv gemm + RoPE + KV write (stream-K)");
    mark_if(mark, 2);
}

void gate_up_swiglu(const SkGemm& g, void* act, cudaStream_t s, const Mark& mark) {
    if (g.path == 0) {
        cuda_check(launch_gemm_streamk(g.tmA, g.tmB, g.M, g.N, g.K, g.sk, s, g.w8), "gate_up gemm (stream-K)"); mark_if(mark, 8);
        cuda_check(launch_sk_swiglu(g.sk, act, g.M, g.N / 2, s), "swiglu"); mark_if(mark, 9);
        return;
    }
    cuda_check(launch_gemm_streamk_swiglu(g.tmA, g.tmB, g.M, g.N / 2, g.K, g.sk, act, g.tile_flags, s, g.w8), "gate_up gemm + SwiGLU (stream-K)");
    mark_if(mark, 8);
}

void step_attention(const CUtensorMap* tm_kv, const KvLayout& kv, DecodeAttnParams dec, PrefillAttnParams pre, int layer, cudaStream_t s,
                    const Mark& mark) {
    dec.layer = pre.layer = layer;
    dec.scale_log2e = pre.scale_log2e = (1.0f / std::sqrt((float)kv.head_dim)) * 1.4426950408889634f;
    if (dec.n_ctas > 0) { cuda_check(launch_decode_attention(tm_kv, kv, dec, s), "decode attention"); mark_if(mark, 4); }
    if (pre.n_tiles > 0) { cuda_check(launch_prefill_attention(tm_kv, kv, pre, s), "prefill attention"); mark_if(mark, 4); }     // mixed step: disjoint rows
}

void lm_head_argmax(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int bn, float* logits, int ldl, float* amax_val,
                    int* amax_idx, const uint32_t* mask_table, const int32_t* mask_slot, int mask_words, int col_offset, int32_t* ids,
                    void* pair_out, cudaStream_t s, const Mark& mark) {
    GemmParams p{}; p.M = M; p.N = N; p.K = K; p.logits = logits; p.ldl = ldl; p.amax_val = amax_val; p.amax_idx = amax_idx;
    p.mask_table = mask_table; p.mask_slot = mask_slot; p.mask_words = mask_words; p.col_offset = col_offset;
    cuda_check(launch_gemm(tmA, tmB, p, EPI_LOGITS, bn, s), "lm_head gemm"); mark_if(mark, 12);
    const int n_tiles = gemm_n_tiles(N, bn);
    if (pair_out) cuda_check(launch_argmax_reduce_pair(amax_val, amax_idx, M, n_tiles, col_offset, pair_out, s), "argmax (local shard)");
    else cuda_check(launch_argmax_reduce(amax_val, amax_idx, M, n_tiles, ids, nullptr, s), "argmax");
}

void proj_gemm(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int epilogue, int bn, void* out, const void* bias,
               const void* resid, W8Scales w8, const char* label, cudaStream_t s) {
    GemmParams p{}; p.M = M; p.N = N; p.K = K; p.out = out; p.ldo = epilogue == EPI_SWIGLU ? N / 2 : N;
    p.bias = bias; p.resid = resid; p.ldr = N; p.w8 = w8;
    cuda_check(launch_gemm(tmA, tmB, p, epilogue, bn, s), label);
}

}  // namespace oa
