// capi_kernels.cpp — kernel-level C entry points on raw device pointers (parity tests drive these with
// torch-allocated memory; nothing here is on the serving path).  The forward's sequences run through its stage functions (stages.hpp).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/opsagent_b200.h"
#include <map>
#include <memory>
#include <mutex>
#include "grammar.hpp"
#include "token_mask.hpp"
#include "model.hpp"
#include "tokenizer.hpp"

using namespace oa;
namespace oa { int fail_host(int code, const std::string& msg); }      // oa_last_error() message (engine.cpp)

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

namespace {
struct DevBuf {
    void* p = nullptr;
    explicit DevBuf(size_t n) { if (cudaMalloc(&p, n ? n : 16) != cudaSuccess) p = nullptr; }
    template <typename T> DevBuf(const T* src, size_t n, cudaStream_t s) : DevBuf(n * sizeof(T)) {      // a copy of n host elements, ordered on s
        if (p && n && cudaMemcpyAsync(p, src, n * sizeof(T), cudaMemcpyHostToDevice, s) != cudaSuccess) { cudaFree(p); p = nullptr; }
    }
    ~DevBuf() { if (p) cudaFree(p); }
};
int rc_of(cudaError_t e) { return e == cudaSuccess ? OA_OK : OA_ERR_INTERNAL; }
// the same, telling a launcher's refusal of its arguments apart from a failed launch
int rc_launch(cudaError_t e) { return e == cudaErrorInvalidValue ? OA_ERR_BAD_REQUEST : rc_of(e); }
// an entry's stage calls, then (sync) the wait for them: the first CUDA error, thrown by a stage or returned by the wait
template <typename F> cudaError_t staged(cudaStream_t s, F&& stages, bool sync = true) {
    try { stages(); } catch (const CudaError& e) { return e.code; }
    return sync ? cudaStreamSynchronize(s) : cudaSuccess;
}

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
// a decode projection entry's maps and stream-K setup (path 0: BLOCK_N block_n, 2 row slots when M > 128; else 128), then stage(g) and the wait
template <typename F> int sk_entry(const void* A, const float* sa, const void* B, const float* sb, int M, int N, int K, int block_n, int n_ctas,
                                   int path, cudaStream_t s, F&& stage) {
    const bool fp8 = sa != nullptr;
    const int bn = path == 0 ? block_n : 128;
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, fp8, M, N, K, bn)) return OA_ERR_INTERNAL;
    SkSetup st(N, K, bn, n_ctas, path == 0 && M > 128 ? 256 : 128, fp8, s);
    if (!st.ok()) return OA_ERR_INTERNAL;
    const SkGemm g{path, &tmA, &tmB, M, N, K, st.sk, W8Scales{sa, sb}, st.tile_flags()};
    return rc_launch(staged(s, [&] { stage(g); }));
}

// one layer of a paged cache: bf16, or with k_scale non-null fp8 with the given scales (k_scale / v_scale point at one float each)
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

int sm_count() { int dev = 0, n = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); return n > 0 ? n : 132; }

// One layer's attention as the engine builds it from host block tables and lengths: decode attention of sequences 0 .. n_decode-1 on the plan
// for n_ctas_target CTAs, then the prefill tiles of the others (q_lens[i] rows each), `launches` times.  merge_inline: the in-kernel merge on
// counters zeroed once (they advance by n_pieces per launch, as per layer in a step); else the separate merge kernel after each launch
int attention(const void* q, void* out, const KvLayout& kv, const int32_t* block_tables, int32_t max_pages_per_seq, const int32_t* ctx_lens,
              const int32_t* q_lens, int32_t n_seqs, int32_t n_decode, int32_t n_heads, int32_t n_ctas_target, int32_t force_splits, bool merge_inline,
              int32_t launches, cudaStream_t s) {
    DecodePlan plan;
    if (n_decode > 0) build_decode_plan(ctx_lens, n_decode, kv.n_kv, n_ctas_target, force_splits, plan);
    std::vector<PrefillTile> tiles;
    for (int i = n_decode, row = n_decode; i < n_seqs; row += q_lens[i++]) append_prefill_tiles(tiles, i, row, ctx_lens[i] - q_lens[i], q_lens[i]);
    sort_prefill_tiles(tiles);
    const size_t slots = (size_t)(plan.n_slots + 1) * (n_heads / kv.n_kv), n_cnt = plan.merges.size() + 1;
    DevBuf bt(block_tables, (size_t)n_seqs * max_pages_per_seq, s), ctx(ctx_lens, (size_t)n_seqs, s), d_tiles(tiles.data(), tiles.size(), s);
    DevBuf segs(plan.segs.data(), plan.segs.size(), s), cta_ptr(plan.cta_ptr.data(), plan.cta_ptr.size(), s), merges(plan.merges.data(), plan.merges.size(), s);
    DevBuf part_o(slots * kv.head_dim * 4), part_ml(slots * 2 * 4), counters(n_cnt * 4);
    CUtensorMap tm;
    if (kv_tmap(&tm, kv) != 0 || !bt.p || !ctx.p || !segs.p || !cta_ptr.p || !merges.p || !d_tiles.p || !part_o.p || !part_ml.p || !counters.p ||
        cudaMemsetAsync(counters.p, 0, n_cnt * 4, s) != cudaSuccess)
        return OA_ERR_INTERNAL;
    const DecodeAttnParams dec{q, out, (const int32_t*)bt.p, (const int32_t*)ctx.p, max_pages_per_seq, (const DecodeSeg*)segs.p, (const int32_t*)cta_ptr.p,
                               (int)plan.cta_ptr.size() - 1, (float*)part_o.p, (float*)part_ml.p, merge_inline ? (int32_t*)counters.p : nullptr, 0, n_heads, kv.n_kv, 0.f};
    const PrefillAttnParams pre{q, out, (const int32_t*)bt.p, max_pages_per_seq, (const PrefillTile*)d_tiles.p, (int)tiles.size(), 0, n_heads, kv.n_kv, 0.f};
    return rc_launch(staged(s, [&] {
        for (int i = 0; i < launches; ++i) {
            step_attention(&tm, kv, dec, pre, 0, s);
            if (!merge_inline)
                cuda_check(launch_decode_merge((const MergeItem*)merges.p, (int)plan.merges.size(), dec.part_o, dec.part_ml, out, n_heads, kv.n_kv, kv.head_dim, s),
                           "decode merge");
        }
    }));
}
int paged_attention(const void* q, void* out, const KvLayout& kv, const int32_t* block_tables, int32_t max_pages_per_seq, const int32_t* ctx_lens,
                    const int32_t* q_lens, int32_t n_seqs, int32_t n_heads, int32_t force_splits, cudaStream_t s) {
    bool decode = true;
    for (int i = 0; i < n_seqs; ++i) if (q_lens && q_lens[i] != 1) decode = false;
    if (decode) return attention(q, out, kv, block_tables, max_pages_per_seq, ctx_lens, nullptr, n_seqs, n_seqs, n_heads, 2 * 132, force_splits, false, 1, s);
    const int rc = attention(q, out, kv, block_tables, max_pages_per_seq, ctx_lens, q_lens, n_seqs, 0, n_heads, 2 * sm_count(), 0, true, 1, s);
    return rc == OA_ERR_BAD_REQUEST ? OA_ERR_INTERNAL : rc;
}
// the engine's RoPE + KV write of a prefill step into one layer of a paged cache
cudaError_t kv_write(const void* qkv, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin, void* q_out,
                     const KvLayout& kv, int32_t T, int32_t n_heads, cudaStream_t s) {
    cudaError_t e = launch_rope_kv_write(qkv, positions, slots, rope_cos, rope_sin, q_out, kv, 0, T, n_heads, s);
    return e == cudaSuccess ? cudaStreamSynchronize(s) : e;
}
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
// the stream-K GEMM of A [M, K] by B [N, K] (bf16, or e4m3 with row scales sa / sb) and the fixed-order sum of its partials -> out_f32 [M, N]
int gemm_streamk_sum(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t block_n,
                     int32_t n_ctas, float* out_f32, cudaStream_t s) {
    const bool fp8 = sa != nullptr;
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, fp8, M, N, K, block_n)) return OA_ERR_INTERNAL;
    DevBuf ws(streamk_ws_bytes(N, block_n, n_ctas, M));
    if (!ws.p) return OA_ERR_INTERNAL;
    const StreamK sk = make_streamk((float*)ws.p, N, K, block_n, n_ctas, M, fp8);
    cudaError_t e = launch_gemm_streamk(&tmA, &tmB, M, N, K, sk, s, W8Scales{sa, sb});
    if (e == cudaSuccess) { sk_reduce_f32_kernel<<<M, 256, 0, s>>>(sk, out_f32, M, N); e = cudaGetLastError(); }
    return rc_of(e == cudaSuccess ? cudaStreamSynchronize(s) : e);
}
}  // namespace

extern "C" {

int oa_k_gemm_streamk(const void* A, const void* B, int32_t M, int32_t N, int32_t K, int32_t block_n, int32_t n_ctas, float* out_f32, void* stream) {
    return gemm_streamk_sum(A, nullptr, B, nullptr, M, N, K, block_n, n_ctas, out_f32, (cudaStream_t)stream);
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
    if (!proj_maps(&tmA, &tmB, A, B, true, M, N, K, block_n)) return OA_ERR_INTERNAL;
    return rc_of(staged(s, [&] { proj_gemm(&tmA, &tmB, M, N, K, epilogue, block_n, out, bias, resid, W8Scales{sa, sb}, "gemm", s); }));
}
// fused: 0 = plain (fp32 out = the fixed-order sum of the partials), 2 = residual add into x [M, N] bf16 (out_f32 unused)
int oa_k_gemm_streamk_fp8(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t block_n,
                          int32_t n_ctas, int32_t fuse, void* x, float* out_f32, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (fuse == 0) return gemm_streamk_sum(A, sa, B, sb, M, N, K, block_n, n_ctas, out_f32, s);
    if (fuse != 2) return OA_ERR_BAD_REQUEST;      // fuse 2 is the residual-add GEMM alone: the forward always follows it with the norm (a stage)
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, true, M, N, K, block_n)) return OA_ERR_INTERNAL;
    SkSetup st(N, K, block_n, n_ctas, M, true, s);
    if (!st.ok()) return OA_ERR_INTERNAL;
    cudaError_t e = launch_gemm_streamk_resid(&tmA, &tmB, M, N, K, st.sk, x, N, st.tile_flags(), s, W8Scales{sa, sb});
    return rc_of(e == cudaSuccess ? cudaStreamSynchronize(s) : e);
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
    if (epilogue == EPI_LOGITS) return oa_k_gemm_logits_masked(A, B, M, N, K, block_n, nullptr, nullptr, 0, 0, logits, argmax_out, stream);
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, false, M, N, K, block_n)) return OA_ERR_INTERNAL;
    cudaStream_t s = (cudaStream_t)stream;
    return rc_of(staged(s, [&] { proj_gemm(&tmA, &tmB, M, N, K, epilogue, block_n, out, bias, resid, W8Scales{}, "gemm", s); }, false));
}

int oa_k_gemm_logits_masked(const void* A, const void* B, int32_t M, int32_t N, int32_t K, int32_t block_n, const uint32_t* mask_table,
                            const int32_t* mask_slot, int32_t mask_words, int32_t col_offset, float* logits, int32_t* ids, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    CUtensorMap tmA, tmB;
    if (!proj_maps(&tmA, &tmB, A, B, false, M, N, K, block_n)) return OA_ERR_INTERNAL;
    const int nt = gemm_n_tiles(N, block_n);
    DevBuf av((size_t)M * nt * 4), ai((size_t)M * nt * 4);
    if (!av.p || !ai.p) return OA_ERR_INTERNAL;
    return rc_launch(staged(s, [&] {
        lm_head_argmax(&tmA, &tmB, M, N, K, block_n, logits, N, (float*)av.p, (int*)ai.p, mask_table, mask_slot, mask_words, col_offset, ids, nullptr, s);
    }));
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
    return rc_of(kv_write(qkv, positions, slots, rope_cos, rope_sin, q_out, one_layer_kv(kv_cache, num_pages, n_kv, head_dim, &k_scale, &v_scale), T,
                          n_heads, (cudaStream_t)stream));
}

int oa_k_kv_write(const void* qkv, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin, void* q_out,
                  void* kv_cache, int32_t num_pages, int32_t T, int32_t n_heads, int32_t n_kv, int32_t head_dim, void* stream) {
    return rc_launch(kv_write(qkv, positions, slots, rope_cos, rope_sin, q_out, one_layer_kv(kv_cache, num_pages, n_kv, head_dim, nullptr, nullptr), T,
                              n_heads, (cudaStream_t)stream));
}

int oa_k_sk_row_parallel(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t block_n,
                         int32_t n_ctas, int32_t path, void* x, const void* gain, void* xn, float eps, int32_t launches, void* stream) {
    if (path < 0 || (path >= 2 && sa)) return OA_ERR_BAD_REQUEST;
    cudaStream_t s = (cudaStream_t)stream;
    return sk_entry(A, sa, B, sb, M, N, K, block_n, n_ctas, path, s, [&](const SkGemm& g) {
        for (int i = 0; i < launches; ++i) finish_row_parallel(g, x, gain, xn, eps, kOProj, s);
    });
}

int oa_k_sk_swiglu(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t F, int32_t K, int32_t block_n,
                   int32_t n_ctas, int32_t path, void* act, int32_t launches, void* stream) {
    if (path != 0 && path != 1) return OA_ERR_BAD_REQUEST;
    cudaStream_t s = (cudaStream_t)stream;
    return sk_entry(A, sa, B, sb, M, 2 * F, K, block_n, n_ctas, path, s, [&](const SkGemm& g) {
        for (int i = 0; i < launches; ++i) gate_up_swiglu(g, act, s);
    });
}

int oa_k_sk_qkv_rope(const void* A, const float* sa, const void* B, const float* sb, const void* bias, int32_t M, int32_t K, int32_t n_heads,
                     int32_t n_kv, int32_t head_dim, int32_t block_n, int32_t n_ctas, int32_t path, const int32_t* positions, const int32_t* slots,
                     const float* rope_cos, const float* rope_sin, void* q_out, void* kv_cache, int32_t num_pages, float k_scale, float v_scale,
                     void* stream) {
    if (path < 0 || (path >= 2 && sa)) return OA_ERR_BAD_REQUEST;
    cudaStream_t s = (cudaStream_t)stream;
    const KvLayout kv = one_layer_kv(kv_cache, num_pages, n_kv, head_dim, k_scale > 0.f ? &k_scale : nullptr, &v_scale);
    return sk_entry(A, sa, B, sb, M, (n_heads + 2 * n_kv) * head_dim, K, block_n, n_ctas, path, s, [&](const SkGemm& g) {
        qkv_rope(g, bias, positions, slots, rope_cos, rope_sin, q_out, kv, 0, n_heads, s);
    });
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
    // the forward's epilogues: bias on the qkv store only, the residual added in place
    return rc_launch(staged(s, [&] {
        proj_gemm(&tmA, &tmB, M, N, K, epilogue, bn, out, epilogue == EPI_STORE ? bias : nullptr, out, W8Scales{sa, sb}, "prefill gemm", s);
    }));
}

int oa_k_step_attention(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables, int32_t max_pages_per_seq,
                        const int32_t* ctx_lens, const int32_t* q_lens, int32_t n_seqs, int32_t n_decode, int32_t n_heads, int32_t n_kv,
                        int32_t head_dim, float k_scale, float v_scale, void* stream) {
    if (n_decode < 0 || n_decode > n_seqs) return OA_ERR_BAD_REQUEST;
    for (int i = 0; i < n_seqs; ++i) if (q_lens[i] < 1 || q_lens[i] > ctx_lens[i] || (i < n_decode && q_lens[i] != 1)) return OA_ERR_BAD_REQUEST;
    return attention(q, out, one_layer_kv(kv_cache, num_pages, n_kv, head_dim, k_scale > 0.f ? &k_scale : nullptr, &v_scale), block_tables,
                     max_pages_per_seq, ctx_lens, q_lens, n_seqs, n_decode, n_heads, 2 * sm_count(), 0, true, 1, (cudaStream_t)stream);
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
    return attention(q, out, one_layer_kv(kv_cache, num_pages, n_kv, head_dim, k_scale > 0.f ? &k_scale : nullptr, &v_scale), block_tables,
                     max_pages_per_seq, ctx_lens, nullptr, n_seqs, n_seqs, n_heads, n_ctas_target, 0, merge_inline != 0, launches, (cudaStream_t)stream);
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
    for (int i = 0; i < launches; ++i) {
        const uint32_t ep = epoch + (uint32_t)i;
        cudaError_t e = staged(s, [&] {
            for (int r = 0; r < t; ++r)
                tp_row_parallel_partial(SkGemm{0, &tmA[r], &tmB[r], M, H, K, st.sk}, bf16_partials != 0, partial[r], signal(r, ep), kOProj, s);
        });
        if (e != cudaSuccess) return rc_launch(e);
        // every consumer below waits for the t signals of this epoch: launch none of them unless all t x t flags already show it
        uint32_t h[TP_MAX * 8];
        if (cudaMemcpy(h, flags, (size_t)t * 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost) != cudaSuccess) return OA_ERR_INTERNAL;
        for (int p = 0; p < t; ++p)
            for (int r = 0; r < t; ++r)
                if (h[p * 8 + r] != ep)
                    return fail_host(OA_ERR_INTERNAL, "tp row-parallel: launch " + std::to_string(i) + ", rank " + std::to_string(r) + " did not signal rank " +
                                                          std::to_string(p) + " (flag " + std::to_string(h[p * 8 + r]) + ", epoch " + std::to_string(ep) + ")");
        e = staged(s, [&] {
            for (int r = 0; r < t; ++r) tp_row_parallel_finish(parts.get(), t, bf16_partials != 0, x[r], gain, xn[r], M, H, eps, signal(r, ep), kOProj, s);
        }, false);
        if (e != cudaSuccess) return rc_launch(e);
    }
    return rc_launch(cudaStreamSynchronize(s));
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
    CUtensorMap tmA, tmB[TP_MAX];
    for (int r = 0; r < t; ++r) if (!proj_maps(&tmA, &tmB[r], A, (const char*)B + (size_t)r * Vs * K * 2, false, M, Vs, K, bn)) return OA_ERR_INTERNAL;
    PeerTable pt(pairs, t);
    DevBuf av((size_t)t * M * nt * 4), ai((size_t)t * M * nt * 4);       // each shard's per-tile (max, arg-max): the engine's amax_val_ / amax_idx_
    if (!pt.get() || !av.p || !ai.p) return OA_ERR_INTERNAL;
    return rc_launch(staged(s, [&] {
        for (int r = 0; r < t; ++r)
            lm_head_argmax(&tmA, &tmB[r], M, Vs, K, bn, logits ? logits + (size_t)r * Vs : nullptr, V, (float*)av.p + (size_t)r * M * nt,
                           (int*)ai.p + (size_t)r * M * nt, mask_table, mask_table ? mask_slot : nullptr, mask_table ? mask_words : 0, r * Vs, nullptr,
                           pairs[r], s);
        cuda_check(launch_ar_argmax(pt.get(), t, M, ids, s), "argmax (all ranks)");
    }));
}

}  // extern "C"

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
