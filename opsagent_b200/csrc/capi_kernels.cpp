// capi_kernels.cpp — kernel-level C entry points on raw device pointers (parity tests drive these with
// torch-allocated memory; nothing here is on the serving path).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/opsagent_b200.h"
#include <map>
#include <memory>
#include <mutex>
#include "grammar.hpp"
#include "token_mask.hpp"
#include "tokenizer.hpp"
#include "model.hpp"
#include "tokenizer.hpp"

using namespace oa;
namespace oa { int fail_host(int code, const std::string& msg); }      // oa_last_error() message (engine.cpp)

namespace {
struct DevBuf {
    void* p = nullptr;
    explicit DevBuf(size_t n) { if (cudaMalloc(&p, n ? n : 16) != cudaSuccess) p = nullptr; }
    ~DevBuf() { if (p) cudaFree(p); }
};
int rc_of(cudaError_t e) { return e == cudaSuccess ? OA_OK : OA_ERR_INTERNAL; }
// the same, telling a launcher's refusal of its arguments apart from a failed launch
int rc_launch(cudaError_t e) { return e == cudaErrorInvalidValue ? OA_ERR_BAD_REQUEST : rc_of(e); }

// A [M, K] and B [N, K] operand maps of a decode projection as the engine builds them: bf16 (boxes {64, 128} / {64, bn}) or, with row
// scales, e4m3 bytes (boxes {128, 128} / {128, bn})
bool proj_maps(CUtensorMap* tmA, CUtensorMap* tmB, const void* A, const void* B, bool fp8, int M, int N, int K, int bn) {
    if (fp8) return make_tmap_u8_2d(tmA, A, (uint64_t)M, (uint64_t)K, 128, 128) == 0 && make_tmap_u8_2d(tmB, B, (uint64_t)N, (uint64_t)K, (uint32_t)bn, 128) == 0;
    return make_tmap_bf16_2d(tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)K, 128, 64) == 0 &&
           make_tmap_bf16_2d(tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)K, (uint32_t)bn, 64) == 0;
}
// one projection's stream-K workspace and zeroed per-tile flags (the engine's sk_ws_ / tile_flags_)
struct SkSetup {
    DevBuf ws, flags; StreamK sk;
    SkSetup(int N, int K, int bn, int G, int rows, bool fp8, cudaStream_t s)
        : ws(streamk_ws_bytes(N, bn, G, rows)), flags((size_t)SK_MAX_FLAG_TILES * 4), sk(make_streamk((float*)ws.p, N, K, bn, G, rows, fp8)) {
        if (flags.p && cudaMemsetAsync(flags.p, 0, (size_t)SK_MAX_FLAG_TILES * 4, s) != cudaSuccess) { cudaFree(flags.p); flags.p = nullptr; }
    }
    bool ok() const { return ws.p && flags.p; }
    unsigned int* tile_flags() const { return (unsigned int*)flags.p; }
};
bool is_cluster_path(int path) { return path >= 2; }

// one layer of a paged cache: bf16, or fp8 with the given scales (k_scale / v_scale point at one float each)
KvLayout one_layer_kv(const void* kv_cache, int32_t num_pages, int32_t n_kv, int32_t head_dim, const float* k_scale, const float* v_scale) {
    KvLayout kv{}; kv.base = const_cast<void*>(kv_cache); kv.page_size = 64; kv.n_kv = n_kv; kv.head_dim = head_dim; kv.num_pages = num_pages;
    kv.kv_stride_rows = (int64_t)num_pages * n_kv * 64; kv.layer_stride_rows = 2 * kv.kv_stride_rows;
    kv.fp8 = k_scale != nullptr; kv.k_scale = k_scale; kv.v_scale = v_scale;
    return kv;
}
int kv_tmap(CUtensorMap* tm, const KvLayout& kv) {
    if (kv.fp8) return make_tmap_u8_2d(tm, kv.base, (uint64_t)kv.layer_stride_rows * kv.head_dim / 128, 128, (uint32_t)(kv.head_dim / 2), 128);
    return make_tmap_bf16_2d(tm, kv.base, (uint64_t)kv.layer_stride_rows, (uint64_t)kv.head_dim, (uint64_t)kv.head_dim, 64, 64);
}

int paged_attention(const void* q, void* out, const KvLayout& kv, const int32_t* block_tables, int32_t max_pages_per_seq, const int32_t* ctx_lens,
                    const int32_t* q_lens, int32_t n_seqs, int32_t n_heads, int32_t force_splits, cudaStream_t s);
int decode_attention(const void* q, void* out, const KvLayout& kv, const int32_t* block_tables, int32_t max_pages_per_seq, const int32_t* ctx_lens,
                     int32_t n_seqs, int32_t n_heads, int32_t n_ctas_target, int32_t force_splits, bool merge_inline, int32_t launches, cudaStream_t s);
int prefill_attention(const void* q, void* out, const KvLayout& kv, const int32_t* block_tables, int32_t max_pages_per_seq, const int32_t* ctx_lens,
                      const int32_t* q_lens, int32_t seq0, int32_t n_seqs, int32_t n_heads, cudaStream_t s);
int sm_count() { int dev = 0, n = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); return n > 0 ? n : 132; }

// A device table of t pointers, the way a tensor-parallel collective reaches its peers' buffers (TpComm's d_peer_sym / d_peer_arg).  On one
// GPU the t entries are t local buffers, and the kernel launched with rank r's arguments does what rank r does on t GPUs.
struct PeerTable {
    void* h[TP_MAX] = {};
    DevBuf d{sizeof(h)};
    PeerTable(const void* const* p, int t, size_t stride = 0) {
        for (int r = 0; r < t; ++r) h[r] = stride ? (char*)const_cast<void*>(p[0]) + r * stride : const_cast<void*>(p[r]);
        if (d.p && cudaMemcpy(d.p, h, sizeof(h), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d.p); d.p = nullptr; }
    }
    void* const* get() const { return (void* const*)d.p; }
};
// the tensor-parallel shapes ModelConfig accepts (config.hpp): 2..8 ranks, rows of a multiple of 8 elements
bool tp_shape_ok(int t, int H) { return t >= 2 && t <= TP_MAX && H > 0 && H % 8 == 0; }
}  // namespace

// test-only: materialise the deterministic fixed-order sum of stream-K partials as fp32 [M,N]
__global__ void sk_reduce_f32_kernel(const StreamK sk, float* __restrict__ out, int M, int N) {
    const int row = blockIdx.x;
    for (int col = threadIdx.x; col < N; col += blockDim.x) {
        const uint32_t tile = (uint32_t)col / (uint32_t)sk.bn, cc = (uint32_t)col - tile * (uint32_t)sk.bn;
        uint32_t c_first, c_last;
        sk_tile_ctas(sk, tile, c_first, c_last);
        float acc = 0.f;
        for (uint32_t c = c_first; c <= c_last; ++c) acc += sk.ws[((size_t)(c + tile) * sk.rows + row) * sk.bn + cc];
        out[(size_t)row * N + col] = acc;
    }
}

extern "C" {

int oa_k_gemm_streamk(const void* A, const void* B, int32_t M, int32_t N, int32_t K, int32_t block_n, int32_t n_ctas, float* out_f32, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    CUtensorMap tmA, tmB;
    if (make_tmap_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)K, 128, 64) != 0) return OA_ERR_INTERNAL;
    if (make_tmap_bf16_2d(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)K, (uint32_t)block_n, 64) != 0) return OA_ERR_INTERNAL;
    DevBuf ws(streamk_ws_bytes(N, block_n, n_ctas, M));
    if (!ws.p) return OA_ERR_INTERNAL;
    StreamK sk = make_streamk((float*)ws.p, N, K, block_n, n_ctas, M);
    cudaError_t e = launch_gemm_streamk(&tmA, &tmB, M, N, K, sk, s);
    if (e == cudaSuccess) { sk_reduce_f32_kernel<<<M, 256, 0, s>>>(sk, out_f32, M, N); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_of(e);
}

int oa_k_quant_rows_e4m3(const void* x, void* q, float* scale, int32_t R, int32_t C, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = launch_quant_rows_e4m3(x, (uint8_t*)q, scale, R, C, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_of(e);
}

// fp8 GEMMs: A [M, K] and B [N, K] e4m3 bytes with fp32 row scales sa [M], sb [N] (device pointers)
int oa_k_gemm_fp8(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t block_n,
                  void* out, const void* bias, const void* resid, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    CUtensorMap tmA, tmB;
    if (make_tmap_u8_2d(&tmA, A, (uint64_t)M, (uint64_t)K, 128, 128) != 0) return OA_ERR_INTERNAL;
    if (make_tmap_u8_2d(&tmB, B, (uint64_t)N, (uint64_t)K, (uint32_t)block_n, 128) != 0) return OA_ERR_INTERNAL;
    GemmParams p{}; p.M = M; p.N = N; p.K = K; p.out = out; p.ldo = epilogue == EPI_SWIGLU ? N / 2 : N;
    p.bias = bias; p.resid = resid; p.ldr = N; p.w8 = W8Scales{sa, sb};
    cudaError_t e = launch_gemm(&tmA, &tmB, p, epilogue, block_n, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_of(e);
}
// fused: 0 = plain (fp32 out = the fixed-order sum of the partials), 2 = residual add into x [M, N] bf16 (out_f32 unused)
int oa_k_gemm_streamk_fp8(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t block_n,
                          int32_t n_ctas, int32_t fuse, void* x, float* out_f32, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    CUtensorMap tmA, tmB;
    if (make_tmap_u8_2d(&tmA, A, (uint64_t)M, (uint64_t)K, 128, 128) != 0) return OA_ERR_INTERNAL;
    if (make_tmap_u8_2d(&tmB, B, (uint64_t)N, (uint64_t)K, (uint32_t)block_n, 128) != 0) return OA_ERR_INTERNAL;
    DevBuf ws(streamk_ws_bytes(N, block_n, n_ctas, M)), flags((size_t)SK_MAX_FLAG_TILES * 4);
    if (!ws.p || !flags.p || cudaMemsetAsync(flags.p, 0, (size_t)SK_MAX_FLAG_TILES * 4, s) != cudaSuccess) return OA_ERR_INTERNAL;
    StreamK sk = make_streamk((float*)ws.p, N, K, block_n, n_ctas, M, true);
    cudaError_t e;
    if (fuse == 2) e = launch_gemm_streamk_resid(&tmA, &tmB, M, N, K, sk, x, N, (unsigned int*)flags.p, s, W8Scales{sa, sb});
    else if (fuse == 0) {
        e = launch_gemm_streamk(&tmA, &tmB, M, N, K, sk, s, W8Scales{sa, sb});
        if (e == cudaSuccess) { sk_reduce_f32_kernel<<<M, 256, 0, s>>>(sk, out_f32, M, N); e = cudaGetLastError(); }
    } else return OA_ERR_BAD_REQUEST;
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_of(e);
}

int oa_k_rmsnorm(const void* x, const void* gain, void* y, int32_t T, int32_t H, float eps, void* stream) {
    return rc_of(launch_rmsnorm(x, gain, y, T, H, eps, (cudaStream_t)stream));
}

int oa_k_init_weight(void* dst, uint64_t seed, uint64_t tensor_id, int64_t tensor_id_b, int64_t rows, int64_t cols, float std,
                     float mean, void* stream) {
    return rc_of(launch_init_weight(dst, seed, tensor_id, tensor_id_b, rows, cols, std, mean, (cudaStream_t)stream));
}

int oa_k_gemm(const void* A, const void* B, int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t block_n, void* out,
              const void* bias, const void* resid, float* logits, int32_t* argmax_out, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    CUtensorMap tmA, tmB;
    if (make_tmap_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)K, 128, 64) != 0) return OA_ERR_INTERNAL;
    if (make_tmap_bf16_2d(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)K, (uint32_t)block_n, 64) != 0) return OA_ERR_INTERNAL;
    GemmParams p{}; p.M = M; p.N = N; p.K = K; p.out = out; p.ldo = epilogue == EPI_SWIGLU ? N / 2 : N;
    p.bias = bias; p.resid = resid; p.ldr = N; p.logits = logits; p.ldl = N;
    if (epilogue == EPI_LOGITS) return oa_k_gemm_logits_masked(A, B, M, N, K, block_n, nullptr, nullptr, 0, 0, logits, argmax_out, stream);
    return rc_of(launch_gemm(&tmA, &tmB, p, epilogue, block_n, s));
}

int oa_k_gemm_logits_masked(const void* A, const void* B, int32_t M, int32_t N, int32_t K, int32_t block_n, const uint32_t* mask_table,
                            const int32_t* mask_slot, int32_t mask_words, int32_t col_offset, float* logits, int32_t* ids, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, false, M, N, K, block_n)) return OA_ERR_INTERNAL;
    const int nt = gemm_n_tiles(N, block_n);
    DevBuf av((size_t)M * nt * 4), ai((size_t)M * nt * 4);
    if (!av.p || !ai.p) return OA_ERR_INTERNAL;
    GemmParams p{}; p.M = M; p.N = N; p.K = K; p.logits = logits; p.ldl = N; p.amax_val = (float*)av.p; p.amax_idx = (int*)ai.p;
    p.mask_table = mask_table; p.mask_slot = mask_slot; p.mask_words = mask_words; p.col_offset = col_offset;
    cudaError_t e = launch_gemm(&tmA, &tmB, p, EPI_LOGITS, block_n, s);
    if (e == cudaSuccess) e = launch_argmax_reduce(p.amax_val, p.amax_idx, M, nt, ids, nullptr, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_paged_attention(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables,
                         int32_t max_pages_per_seq, const int32_t* ctx_lens, const int32_t* q_lens, int32_t n_seqs,
                         int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t force_splits, void* stream) {
    return paged_attention(q, out, one_layer_kv(kv_cache, num_pages, n_kv, head_dim, nullptr, nullptr), block_tables, max_pages_per_seq, ctx_lens,
                           q_lens, n_seqs, n_heads, force_splits, (cudaStream_t)stream);
}

int oa_k_paged_attention_fp8(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables,
                             int32_t max_pages_per_seq, const int32_t* ctx_lens, const int32_t* q_lens, int32_t n_seqs,
                             int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t force_splits, float k_scale, float v_scale, void* stream) {
    return paged_attention(q, out, one_layer_kv(kv_cache, num_pages, n_kv, head_dim, &k_scale, &v_scale), block_tables, max_pages_per_seq, ctx_lens,
                           q_lens, n_seqs, n_heads, force_splits, (cudaStream_t)stream);
}

int oa_k_kv_write_fp8(const void* qkv, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin, void* q_out,
                      void* kv_cache, int32_t num_pages, int32_t T, int32_t n_heads, int32_t n_kv, int32_t head_dim, float k_scale, float v_scale,
                      void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const KvLayout kv = one_layer_kv(kv_cache, num_pages, n_kv, head_dim, &k_scale, &v_scale);
    cudaError_t e = launch_rope_kv_write(qkv, positions, slots, rope_cos, rope_sin, q_out, kv, 0, T, n_heads, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_of(e);
}

int oa_k_kv_write(const void* qkv, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin, void* q_out,
                  void* kv_cache, int32_t num_pages, int32_t T, int32_t n_heads, int32_t n_kv, int32_t head_dim, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const KvLayout kv = one_layer_kv(kv_cache, num_pages, n_kv, head_dim, nullptr, nullptr);
    cudaError_t e = launch_rope_kv_write(qkv, positions, slots, rope_cos, rope_sin, q_out, kv, 0, T, n_heads, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_sk_row_parallel(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t block_n,
                         int32_t n_ctas, int32_t path, void* x, const void* gain, void* xn, float eps, int32_t launches, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const bool fp8 = sa != nullptr, ck = is_cluster_path(path);
    if (path < 0 || (ck && fp8)) return OA_ERR_BAD_REQUEST;
    const int bn = path == 0 ? block_n : 128;
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, fp8, M, N, K, bn)) return OA_ERR_INTERNAL;
    SkSetup st(N, K, bn, n_ctas, path == 0 && M > 128 ? 256 : 128, fp8, s);
    if (!st.ok()) return OA_ERR_INTERNAL;
    const W8Scales w8{sa, sb};
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < launches && e == cudaSuccess; ++i) {
        if (path == 0) {
            e = launch_gemm_streamk(&tmA, &tmB, M, N, K, st.sk, s, w8);
            if (e == cudaSuccess) e = launch_sk_resid_rmsnorm(st.sk, x, gain, xn, M, N, eps, s);
            continue;
        }
        e = ck ? launch_gemm_clusterk_resid(&tmA, &tmB, M, N, K, path, x, N, s)
               : launch_gemm_streamk_resid(&tmA, &tmB, M, N, K, st.sk, x, N, st.tile_flags(), s, w8);
        if (e == cudaSuccess) e = launch_rmsnorm_wide(x, gain, xn, M, N, eps, s);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_sk_swiglu(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t F, int32_t K, int32_t block_n,
                   int32_t n_ctas, int32_t path, void* act, int32_t launches, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const bool fp8 = sa != nullptr;
    if (path != 0 && path != 1) return OA_ERR_BAD_REQUEST;
    const int bn = path == 0 ? block_n : 128;
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, fp8, M, 2 * F, K, bn)) return OA_ERR_INTERNAL;
    SkSetup st(2 * F, K, bn, n_ctas, path == 0 && M > 128 ? 256 : 128, fp8, s);
    if (!st.ok()) return OA_ERR_INTERNAL;
    const W8Scales w8{sa, sb};
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < launches && e == cudaSuccess; ++i) {
        if (path == 0) {
            e = launch_gemm_streamk(&tmA, &tmB, M, 2 * F, K, st.sk, s, w8);
            if (e == cudaSuccess) e = launch_sk_swiglu(st.sk, act, M, F, s);
        } else {
            e = launch_gemm_streamk_swiglu(&tmA, &tmB, M, F, K, st.sk, act, st.tile_flags(), s, w8);
        }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_sk_qkv_rope(const void* A, const float* sa, const void* B, const float* sb, const void* bias, int32_t M, int32_t K, int32_t n_heads,
                     int32_t n_kv, int32_t head_dim, int32_t block_n, int32_t n_ctas, int32_t path, const int32_t* positions, const int32_t* slots,
                     const float* rope_cos, const float* rope_sin, void* q_out, void* kv_cache, int32_t num_pages, float k_scale, float v_scale,
                     void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const bool fp8 = sa != nullptr, ck = is_cluster_path(path);
    if (path < 0 || (ck && fp8)) return OA_ERR_BAD_REQUEST;
    const int N = (n_heads + 2 * n_kv) * head_dim, bn = path == 0 ? block_n : 128;
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, fp8, M, N, K, bn)) return OA_ERR_INTERNAL;
    SkSetup st(N, K, bn, n_ctas, path == 0 && M > 128 ? 256 : 128, fp8, s);
    if (!st.ok()) return OA_ERR_INTERNAL;
    const bool kv8 = k_scale > 0.f;
    const KvLayout kv = one_layer_kv(kv_cache, num_pages, n_kv, head_dim, kv8 ? &k_scale : nullptr, kv8 ? &v_scale : nullptr);
    const SkRopeArgs rope = make_sk_rope_args(bias, positions, slots, rope_cos, rope_sin, q_out, kv, 0, n_heads);
    cudaError_t e;
    if (path == 0) {
        e = launch_gemm_streamk(&tmA, &tmB, M, N, K, st.sk, s, W8Scales{sa, sb});
        if (e == cudaSuccess) e = launch_sk_rope_kv_write(st.sk, bias, positions, slots, rope_cos, rope_sin, q_out, kv, 0, M, n_heads, s);
    } else if (ck) {
        e = launch_gemm_clusterk_rope(&tmA, &tmB, M, N, K, path, rope, s);
    } else {
        e = launch_gemm_streamk_rope(&tmA, &tmB, M, N, K, st.sk, rope, st.tile_flags(), s, W8Scales{sa, sb});
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_prefill_gemm(const void* A, const float* sa, const void* B, const float* sb, int32_t a_rows, int32_t M, int32_t N, int32_t K, int32_t epilogue,
                      int32_t block_n, void* out, const void* bias, int32_t* block_n_used, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const bool fp8 = sa != nullptr;
    if (a_rows < M || epilogue < EPI_STORE || epilogue > EPI_SWIGLU) return OA_ERR_BAD_REQUEST;
    const int bn = block_n ? block_n : pick_bn(M, N, sm_count(), 0, fp8);
    if (block_n_used) *block_n_used = bn;
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, fp8, a_rows, N, K, bn)) return OA_ERR_INTERNAL;
    GemmParams p{}; p.M = M; p.N = N; p.K = K; p.out = out; p.ldo = epilogue == EPI_SWIGLU ? N / 2 : N;
    if (epilogue == EPI_STORE) p.bias = bias;
    if (epilogue == EPI_RESID) { p.resid = out; p.ldr = N; }
    p.w8 = W8Scales{sa, sb};
    cudaError_t e = launch_gemm(&tmA, &tmB, p, epilogue, bn, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_step_attention(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables, int32_t max_pages_per_seq,
                        const int32_t* ctx_lens, const int32_t* q_lens, int32_t n_seqs, int32_t n_decode, int32_t n_heads, int32_t n_kv,
                        int32_t head_dim, float k_scale, float v_scale, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n_decode < 0 || n_decode > n_seqs) return OA_ERR_BAD_REQUEST;
    for (int i = 0; i < n_seqs; ++i) if (q_lens[i] < 1 || q_lens[i] > ctx_lens[i] || (i < n_decode && q_lens[i] != 1)) return OA_ERR_BAD_REQUEST;
    const bool kv8 = k_scale > 0.f;
    const KvLayout kv = one_layer_kv(kv_cache, num_pages, n_kv, head_dim, kv8 ? &k_scale : nullptr, kv8 ? &v_scale : nullptr);
    if (n_decode > 0) {
        const int rc = decode_attention(q, out, kv, block_tables, max_pages_per_seq, ctx_lens, n_decode, n_heads, 2 * sm_count(), 0, true, 1, s);
        if (rc != OA_OK) return rc;
    }
    if (n_decode == n_seqs) return OA_OK;
    return prefill_attention(q, out, kv, block_tables, max_pages_per_seq, ctx_lens, q_lens, n_decode, n_seqs, n_heads, s);
}

int oa_k_embed_gather(const int32_t* ids, const void* table, void* out, int32_t T, int32_t H, int32_t vocab, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = launch_embed_gather(ids, table, out, T, H, vocab, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_decode_attention(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables, int32_t max_pages_per_seq,
                          const int32_t* ctx_lens, int32_t n_seqs, int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t n_ctas_target,
                          int32_t merge_inline, int32_t launches, float k_scale, float v_scale, void* stream) {
    const bool kv8 = k_scale > 0.f;
    return decode_attention(q, out, one_layer_kv(kv_cache, num_pages, n_kv, head_dim, kv8 ? &k_scale : nullptr, kv8 ? &v_scale : nullptr), block_tables,
                            max_pages_per_seq, ctx_lens, n_seqs, n_heads, n_ctas_target, 0, merge_inline != 0, launches, (cudaStream_t)stream);
}

// ---- the tensor-parallel collectives, t ranks emulated one after another on one stream (see the header) ----
int oa_k_tp_row_parallel(int32_t t, const void* const* A, const void* const* B, int32_t M, int32_t H, int32_t K, int32_t block_n, int32_t n_ctas,
                         int32_t bf16_partials, void* const* partial, void* const* x, void* const* xn, const void* gain, float eps, uint32_t* flags,
                         uint32_t epoch, int32_t launches, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!tp_shape_ok(t, H) || M <= 0 || launches < 1) return OA_ERR_BAD_REQUEST;
    CUtensorMap tmA[TP_MAX], tmB[TP_MAX];
    for (int r = 0; r < t; ++r) if (!proj_maps(&tmA[r], &tmB[r], A[r], B[r], false, M, H, K, block_n)) return OA_ERR_INTERNAL;
    // one workspace for every rank: rank r + 1's GEMM runs after rank r's reduce in stream order
    SkSetup st(H, K, block_n, n_ctas, M > 128 ? 256 : 128, false, s);
    DevBuf done((size_t)TP_MAX * 64);                     // each rank's "CTAs finished" counter, on its own 64 bytes as TpComm allocates it
    const void* fbase = flags;
    PeerTable parts(partial, t), peer_flags(&fbase, t, 8 * sizeof(uint32_t));
    if (!st.ok() || !done.p || !parts.get() || !peer_flags.get() || cudaMemsetAsync(done.p, 0, (size_t)TP_MAX * 64, s) != cudaSuccess) return OA_ERR_INTERNAL;
    auto signal = [&](int r, uint32_t e) {
        return TpComm::Signal{(uint32_t* const*)peer_flags.get(), flags + r * 8, (unsigned int*)done.p + r * 16, r, t, e};
    };
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < launches; ++i) {
        const uint32_t ep = epoch + (uint32_t)i;
        for (int r = 0; r < t && e == cudaSuccess; ++r) {
            const TpComm::Signal sg = signal(r, ep);
            e = launch_gemm_streamk(&tmA[r], &tmB[r], M, H, K, st.sk, s);
            if (e == cudaSuccess)
                e = bf16_partials ? launch_sk_reduce_bf16(st.sk, partial[r], M, H, s, &sg) : launch_sk_reduce_f32(st.sk, (float*)partial[r], M, H, s, &sg);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) return rc_launch(e);
        // every consumer below waits for the t signals of this epoch: launch none of them unless all t x t flags already show it
        uint32_t h[TP_MAX * 8];
        if (cudaMemcpy(h, flags, (size_t)t * 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost) != cudaSuccess) return OA_ERR_INTERNAL;
        for (int p = 0; p < t; ++p)
            for (int r = 0; r < t; ++r)
                if (h[p * 8 + r] != ep)
                    return fail_host(OA_ERR_INTERNAL, "tp row-parallel: launch " + std::to_string(i) + ", rank " + std::to_string(r) + " did not signal rank " +
                                                          std::to_string(p) + " (flag " + std::to_string(h[p * 8 + r]) + ", epoch " + std::to_string(ep) + ")");
        for (int r = 0; r < t && e == cudaSuccess; ++r) {
            const TpComm::Signal sg = signal(r, ep);
            e = bf16_partials ? launch_ar_resid_rmsnorm_bf16in(parts.get(), t, x[r], gain, xn[r], M, H, eps, s, &sg)
                              : launch_ar_resid_rmsnorm(parts.get(), t, x[r], gain, xn[r], M, H, eps, s, &sg);
        }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_tp_allreduce_prefill(int32_t t, void* const* partial, void* const* x, void* const* gather, int32_t T, int32_t H, int32_t two_shot, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!tp_shape_ok(t, H) || T < 0 || (two_shot && !gather)) return OA_ERR_BAD_REQUEST;
    PeerTable parts(partial, t);
    if (!parts.get()) return OA_ERR_INTERNAL;
    cudaError_t e = cudaSuccess;
    if (!two_shot) {
        for (int r = 0; r < t && e == cudaSuccess; ++r) e = launch_ar_resid_bf16(parts.get(), t, x[r], T, H, s);
    } else {                                              // stream order stands in for the engine's barrier between the two halves
        PeerTable gath(gather, t);
        if (!gath.get()) return OA_ERR_INTERNAL;
        for (int r = 0; r < t && e == cudaSuccess; ++r) e = launch_ar2_reduce_scatter(parts.get(), t, r, x[r], gather[r], T, H, s);
        for (int r = 0; r < t && e == cudaSuccess; ++r) e = launch_ar2_all_gather(gath.get(), t, r, x[r], T, H, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);      // before gath's table is freed
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

int oa_k_tp_lm_head_argmax(int32_t t, const void* A, const void* B, int32_t M, int32_t V, int32_t K, int32_t block_n, const uint32_t* mask_table,
                           const int32_t* mask_slot, int32_t mask_words, float* logits, void* const* pairs, int32_t* ids, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!tp_shape_ok(t, K) || M <= 0 || V <= 0 || V % t || (V / t) % 8) return OA_ERR_BAD_REQUEST;
    const int Vs = V / t, bn = block_n ? block_n : pick_bn(M, Vs, sm_count(), 0), nt = gemm_n_tiles(Vs, bn);
    PeerTable pt(pairs, t);
    DevBuf av((size_t)t * M * nt * 4), ai((size_t)t * M * nt * 4);       // each shard's per-tile (max, arg-max): the engine's amax_val_ / amax_idx_
    if (!pt.get() || !av.p || !ai.p) return OA_ERR_INTERNAL;
    cudaError_t e = cudaSuccess;
    for (int r = 0; r < t && e == cudaSuccess; ++r) {
        CUtensorMap tmA, tmB;
        if (!proj_maps(&tmA, &tmB, A, (const char*)B + (size_t)r * Vs * K * 2, false, M, Vs, K, bn)) return OA_ERR_INTERNAL;
        GemmParams p{}; p.M = M; p.N = Vs; p.K = K; p.logits = logits ? logits + (size_t)r * Vs : nullptr; p.ldl = V;
        p.amax_val = (float*)av.p + (size_t)r * M * nt; p.amax_idx = (int*)ai.p + (size_t)r * M * nt;
        if (mask_table) { p.mask_table = mask_table; p.mask_slot = mask_slot; p.mask_words = mask_words; p.col_offset = r * Vs; }
        e = launch_gemm(&tmA, &tmB, p, EPI_LOGITS, bn, s);
        if (e == cudaSuccess) e = launch_argmax_reduce_pair(p.amax_val, p.amax_idx, M, nt, r * Vs, pairs[r], s);
    }
    if (e == cudaSuccess) e = launch_ar_argmax(pt.get(), t, M, ids, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

}  // extern "C"

namespace {
int paged_attention(const void* q, void* out, const KvLayout& kv, const int32_t* block_tables, int32_t max_pages_per_seq, const int32_t* ctx_lens,
                    const int32_t* q_lens, int32_t n_seqs, int32_t n_heads, int32_t force_splits, cudaStream_t s) {
    bool decode = true;
    for (int i = 0; i < n_seqs; ++i) if (q_lens && q_lens[i] != 1) decode = false;
    if (decode) return decode_attention(q, out, kv, block_tables, max_pages_per_seq, ctx_lens, n_seqs, n_heads, 2 * 132, force_splits, false, 1, s);
    const int rc = prefill_attention(q, out, kv, block_tables, max_pages_per_seq, ctx_lens, q_lens, 0, n_seqs, n_heads, s);
    return rc == OA_ERR_BAD_REQUEST ? OA_ERR_INTERNAL : rc;
}

// prefill attention of sequences seq0 .. n_seqs-1 (q_lens[i] new rows each, after the sum of q_lens[0 .. seq0-1] rows of the token batch):
// their 128-row tiles, built and ordered as the engine's prefill step builds and orders them
int prefill_attention(const void* q, void* out, const KvLayout& kv, const int32_t* block_tables, int32_t max_pages_per_seq, const int32_t* ctx_lens,
                      const int32_t* q_lens, int32_t seq0, int32_t n_seqs, int32_t n_heads, cudaStream_t s) {
    CUtensorMap tm;
    if (kv_tmap(&tm, kv) != 0) return OA_ERR_INTERNAL;
    const float scale_log2e = (1.0f / std::sqrt((float)kv.head_dim)) * 1.4426950408889634f;
    std::vector<PrefillTile> tiles; int row = 0;
    for (int i = 0; i < seq0; ++i) row += q_lens[i];
    for (int i = seq0; i < n_seqs; ++i) {
        append_prefill_tiles(tiles, i, row, ctx_lens[i] - q_lens[i], q_lens[i]);
        row += q_lens[i];
    }
    sort_prefill_tiles(tiles);
    DevBuf d_bt((size_t)n_seqs * max_pages_per_seq * 4), d_tiles(tiles.size() * sizeof(PrefillTile));
    if (!d_bt.p || !d_tiles.p) return OA_ERR_INTERNAL;
    cudaMemcpyAsync(d_bt.p, block_tables, (size_t)n_seqs * max_pages_per_seq * 4, cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_tiles.p, tiles.data(), tiles.size() * sizeof(PrefillTile), cudaMemcpyHostToDevice, s);
    PrefillAttnParams a{}; a.q = q; a.out = out; a.block_tables = (const int32_t*)d_bt.p; a.max_pages_per_seq = max_pages_per_seq;
    a.tiles = (const PrefillTile*)d_tiles.p; a.n_tiles = (int)tiles.size(); a.layer = 0; a.n_heads = n_heads; a.n_kv = kv.n_kv; a.scale_log2e = scale_log2e;
    cudaError_t e = launch_prefill_attention(&tm, kv, a, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}

// one decode-attention step on build_decode_plan's work plan.  merge_inline: the engine's in-kernel merge, on counters zeroed once and carried
// across `launches` launches (they advance by n_pieces per launch, as per layer in a step); else the separate merge kernel after each launch
int decode_attention(const void* q, void* out, const KvLayout& kv, const int32_t* block_tables, int32_t max_pages_per_seq, const int32_t* ctx_lens,
                     int32_t n_seqs, int32_t n_heads, int32_t n_ctas_target, int32_t force_splits, bool merge_inline, int32_t launches, cudaStream_t s) {
    const int n_kv = kv.n_kv, head_dim = kv.head_dim, grp = n_heads / n_kv;
    CUtensorMap tm;
    if (kv_tmap(&tm, kv) != 0) return OA_ERR_INTERNAL;
    DecodePlan plan;
    build_decode_plan(ctx_lens, n_seqs, n_kv, n_ctas_target, force_splits, plan);
    DevBuf d_bt((size_t)n_seqs * max_pages_per_seq * 4), d_ctx((size_t)n_seqs * 4);
    DevBuf d_segs(plan.segs.size() * sizeof(DecodeSeg)), d_ptr(plan.cta_ptr.size() * 4), d_merge(plan.merges.size() * sizeof(MergeItem));
    DevBuf d_po((size_t)(plan.n_slots + 1) * grp * head_dim * 4), d_pml((size_t)(plan.n_slots + 1) * grp * 2 * 4), d_cnt((plan.merges.size() + 1) * 4);
    if (!d_bt.p || !d_ctx.p || !d_segs.p || !d_ptr.p || !d_merge.p || !d_po.p || !d_pml.p || !d_cnt.p) return OA_ERR_INTERNAL;
    cudaMemcpyAsync(d_bt.p, block_tables, (size_t)n_seqs * max_pages_per_seq * 4, cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_ctx.p, ctx_lens, (size_t)n_seqs * 4, cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_segs.p, plan.segs.data(), plan.segs.size() * sizeof(DecodeSeg), cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_ptr.p, plan.cta_ptr.data(), plan.cta_ptr.size() * 4, cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_merge.p, plan.merges.data(), plan.merges.size() * sizeof(MergeItem), cudaMemcpyHostToDevice, s);
    cudaMemsetAsync(d_cnt.p, 0, (plan.merges.size() + 1) * 4, s);
    DecodeAttnParams a{}; a.q = q; a.out = out; a.block_tables = (const int32_t*)d_bt.p; a.ctx_lens = (const int32_t*)d_ctx.p;
    a.max_pages_per_seq = max_pages_per_seq; a.segs = (const DecodeSeg*)d_segs.p; a.cta_seg_ptr = (const int32_t*)d_ptr.p;
    a.n_ctas = (int)plan.cta_ptr.size() - 1; a.part_o = (float*)d_po.p; a.part_ml = (float*)d_pml.p; a.layer = 0;
    a.merge_counters = merge_inline ? (int32_t*)d_cnt.p : nullptr;
    a.n_heads = n_heads; a.n_kv = n_kv; a.scale_log2e = (1.0f / std::sqrt((float)head_dim)) * 1.4426950408889634f;
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < launches && e == cudaSuccess; ++i) {
        e = launch_decode_attention(&tm, kv, a, s);
        if (e == cudaSuccess && !merge_inline)
            e = launch_decode_merge((const MergeItem*)d_merge.p, (int)plan.merges.size(), a.part_o, a.part_ml, out, n_heads, n_kv, head_dim, s);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return rc_launch(e);
}
}  // namespace

extern "C" {


int oa_host_apply_chat_template(const char* config_json, const oa_msg* msgs, int32_t n_msgs, int32_t* out_ids, int32_t cap, int32_t* n_out) {
    try {
        ModelConfig mc; EngineOptions eo; parse_config(config_json ? config_json : "{}", mc, eo);
        Tokenizer tok(mc, eo.tokenizer);
        std::vector<ChatMessage> m;
        for (int i = 0; i < n_msgs; ++i) m.push_back(ChatMessage{msgs[i].role, msgs[i].content});
        auto ids = tok.apply_chat_template(m);
        *n_out = (int32_t)ids.size();
        if (out_ids) std::memcpy(out_ids, ids.data(), (size_t)std::min<int32_t>(cap, (int32_t)ids.size()) * 4);
    } catch (const std::exception&) { return OA_ERR_BAD_REQUEST; }
    return OA_OK;
}

int oa_host_decode_plan(const int32_t* ctx_lens, int32_t n_seqs, int32_t n_kv, int32_t n_ctas_target, int32_t force_splits,
                        int32_t* segs_out, int32_t cap_segs, int32_t* cta_ptr_out, int32_t cap_ctas, int32_t* n_ctas_out,
                        int32_t* n_segs_out, int32_t* n_slots_out) {
    DecodePlan plan;
    build_decode_plan(ctx_lens, n_seqs, n_kv, n_ctas_target, force_splits, plan);
    if ((int)plan.segs.size() > cap_segs || (int)plan.cta_ptr.size() > cap_ctas + 1) return OA_ERR_BAD_REQUEST;
    for (size_t i = 0; i < plan.segs.size(); ++i) {
        const DecodeSeg& g = plan.segs[i];
        int32_t* o = segs_out + i * 5; o[0] = g.seq; o[1] = g.kvh; o[2] = g.chunk_begin; o[3] = g.chunk_end; o[4] = g.partial_slot;
    }
    std::memcpy(cta_ptr_out, plan.cta_ptr.data(), plan.cta_ptr.size() * 4);
    *n_ctas_out = (int32_t)plan.cta_ptr.size() - 1; *n_segs_out = (int32_t)plan.segs.size(); *n_slots_out = plan.n_slots;
    return OA_OK;
}

int oa_host_streamk_plan(int32_t N, int32_t K, int32_t block_n, int32_t n_ctas, int64_t* cta_unit0_out, int32_t cap_ctas,
                         int32_t* tile_first_out, int32_t* tile_last_out, int32_t cap_tiles, int32_t* n_ctas_out, int32_t* n_tiles_out,
                         int32_t* kb_out) {
    if (N <= 0 || K <= 0 || n_ctas <= 0 || (block_n != 128 && block_n != 256)) return OA_ERR_BAD_REQUEST;
    const StreamK sk = make_streamk(nullptr, N, K, block_n, n_ctas);
    if (sk.G > cap_ctas || sk.n_tiles > cap_tiles) return OA_ERR_BAD_REQUEST;
    for (int c = 0; c <= sk.G; ++c) cta_unit0_out[c] = (long long)c * sk.total / sk.G;            // the kernels' u0/u1
    for (int t = 0; t < sk.n_tiles; ++t) {                                                        // the very function the kernels call
        uint32_t cf, cl;
        sk_tile_ctas(sk, (uint32_t)t, cf, cl);
        tile_first_out[t] = (int32_t)cf; tile_last_out[t] = (int32_t)cl;
    }
    *n_ctas_out = sk.G; *n_tiles_out = sk.n_tiles; *kb_out = sk.kb;
    return OA_OK;
}

int32_t oa_host_pick_bn(int32_t M, int32_t N, int32_t sm_count, int32_t override_bn, int32_t fp8) {
    return pick_bn(M, N, sm_count, override_bn, fp8 != 0);
}

int oa_host_grammar_step(int32_t kind, const uint8_t* prefix, int32_t n, uint32_t* mask_out, int32_t* done_out) {
    return oa_host_grammar_step_ex(kind, "", prefix, n, mask_out, done_out);
}
int oa_host_grammar_step_ex(int32_t kind, const char* functions, const uint8_t* prefix, int32_t n, uint32_t* mask_out, int32_t* done_out) {
    if (kind < GRAMMAR_TOOLCALL || kind > GRAMMAR_TEXT) return OA_ERR_BAD_REQUEST;
    ToolPromptGrammar g(kind, functions ? functions : "");
    if (!g.active()) return OA_ERR_BAD_REQUEST;
    for (int i = 0; i < n; ++i) if (!g.advance(prefix[i])) return OA_ERR_BAD_REQUEST;
    g.allowed(mask_out); *done_out = g.done() ? 1 : 0;
    return OA_OK;
}

int oa_host_grammar_token_mask(const char* tokenizer_json_path, int32_t vocab, int32_t kind, const char* functions, const uint8_t* prefix, int32_t n,
                               uint32_t* mask_out, int32_t cap_words, char* key_out, int32_t key_cap) {
    if (kind < GRAMMAR_TOOLCALL || kind > GRAMMAR_TEXT || vocab <= 0 || !mask_out) return OA_ERR_BAD_REQUEST;
    try {
        // one trie per (tokenizer, vocab), built once: the same structure the engine builds at start-up
        static std::mutex mu; static std::map<std::string, std::shared_ptr<TokenTrie>> tries;
        const std::string tk = std::string(tokenizer_json_path ? tokenizer_json_path : "") + "#" + std::to_string(vocab);
        std::shared_ptr<TokenTrie> trie;
        {
            std::lock_guard<std::mutex> lk(mu);
            auto it = tries.find(tk);
            if (it == tries.end()) {
                ModelConfig mc; mc.vocab = vocab; mc.chat_template = "llama3";
                std::vector<std::string> bytes;
                if (tokenizer_json_path && tokenizer_json_path[0]) bytes = BpeTokenizer::load(tokenizer_json_path)->text_token_bytes();
                else { bytes.resize(256); for (int b = 0; b < 256; ++b) bytes[b] = std::string(1, (char)b); }
                trie = std::make_shared<TokenTrie>(); trie->build(bytes, vocab); tries[tk] = trie;
            } else trie = it->second;
        }
        if (trie->words() > cap_words) return OA_ERR_BAD_REQUEST;
        ToolPromptGrammar g(kind, functions ? functions : "");
        if (!g.active()) return OA_ERR_BAD_REQUEST;
        for (int i = 0; i < n; ++i) if (!g.advance(prefix[i])) return OA_ERR_BAD_REQUEST;
        trie->allowed_tokens(g, g.cursor(), mask_out);
        if (key_out && key_cap > 0) std::snprintf(key_out, (size_t)key_cap, "%s", grammar_mask_key(g, g.cursor()).c_str());
    } catch (const std::exception&) { return OA_ERR_BAD_REQUEST; }
    return OA_OK;
}

int oa_host_model_info(const char* config_json, char* buf, size_t n) {
    try {
        ModelConfig c; EngineOptions eo; parse_config(config_json ? config_json : "{}", c, eo);
        std::snprintf(buf, n, "{\"model\": \"%s\", \"hidden\": %d, \"n_layers\": %d, \"n_heads\": %d, \"n_kv_heads\": %d, \"head_dim\": %d, "
                      "\"ffn\": %d, \"vocab\": %d, \"tie_embeddings\": %d, \"qkv_bias\": %d, \"rope_scaling\": %d, \"rope_theta\": %.1f, "
                      "\"rms_eps\": %g, \"template\": \"%s\", \"decode_weight_bytes\": %.0f, \"kv_bytes_per_token\": %zu%s%s}",
                      c.name.c_str(), c.hidden, c.n_layers, c.n_heads, c.n_kv_heads, c.head_dim, c.ffn, c.vocab, c.tie_embeddings, c.qkv_bias,
                      c.rope_scaling, c.rope_theta, c.rms_eps, c.chat_template.c_str(), c.decode_weight_bytes(), c.kv_bytes_per_token(),
                      c.kv_fp8() ? ", \"kv_cache_dtype\": \"fp8_e4m3\"" : "", c.w_fp8() ? ", \"weight_dtype\": \"fp8_e4m3\"" : "");
    } catch (const std::exception& e) { return fail_host(OA_ERR_BAD_REQUEST, e.what()); }
    return OA_OK;
}

}  // extern "C"
