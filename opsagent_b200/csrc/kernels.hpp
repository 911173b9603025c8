// kernels.hpp — host-side launch API of the sm_90a kernels (csrc/*.cu).  Device pointers in,
// cudaError_t out; every launcher is asynchronous on the given stream.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace oa {


// ---- TMA descriptors (tma.cpp) --------------------------------------------------------------
// 2D row-major bf16 tensor [rows, cols] with row pitch `pitch_elems`; box = {box_cols(<=64), box_rows(<=256)},
// 128-byte swizzle.  Returns 0 on success (driver entry point resolved through the runtime, no -lcuda).
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems,
                      uint32_t box_rows, uint32_t box_cols);
// 2D row-major byte tensor [rows, cols] (dense rows), box = {box_cols(<=128), box_rows(<=256)}, 128-byte swizzle (the fp8 KV pool)
int make_tmap_u8_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols);

// ---- GEMM (gemm_wgmma.cu): C[M,N] = A[M,K] . B[N,K]^T, bf16 in, fp32 accumulate in registers ----
enum GemmEpilogue : int {
    EPI_STORE = 0,    // out[M,N] bf16 = acc (+ bias[N])
    EPI_RESID = 1,    // out[M,N] bf16 = acc + resid[M,N]      (out may alias resid)
    EPI_SWIGLU = 2,   // out[M,N/2] bf16 = silu(gate)*up, B rows interleaved 16 gate / 16 up
    EPI_LOGITS = 3,   // per-row (max, argmax) partial per N-tile -> argmax_ws; optional fp32 logits store
};
// fp8 (e4m3) operands: A[M,K] and B[N,K] hold bytes, and C[m,n] = a[m] * b[n] * sum_k A[m,k] B[n,k] with the fp32 row scales a[M], b[N]
// (the quantiser below).  Both null: bf16 operands.
struct W8Scales { const float* a; const float* b; };
struct GemmParams {
    int M, N, K;
    void* out; int ldo;             // bf16 output, leading dimension in elements
    const void* bias;               // bf16 [N] or null        (EPI_STORE)
    const void* resid; int ldr;     // bf16 [M, ldr]           (EPI_RESID)
    float* logits; int ldl;         // optional fp32 [M, ldl]  (EPI_LOGITS)
    float* amax_val; int* amax_idx; // [M, n_tiles]            (EPI_LOGITS)
    // grammar-constrained rows (EPI_LOGITS): row r with mask_slot[r] >= 0 takes its arg-max only over the token ids whose bit is set in
    // mask_table[mask_slot[r] * mask_words ...]; bit index = col_offset + column (col_offset: first global id of a vocab-parallel shard)
    const uint32_t* mask_table; const int32_t* mask_slot; int mask_words, col_offset;
    W8Scales w8;                    // fp8 operands (EPI_STORE / EPI_RESID / EPI_SWIGLU, block_n <= 128)
};
// tmA: box {64, 128} over A[M,K]; tmB: box {64, block_n} over B[N,K].  block_n in {32,64,128,256}.  fp8: byte maps (make_tmap_u8_2d) with
// boxes {128, 128} and {128, block_n}.
cudaError_t launch_gemm(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, int epilogue, int block_n,
                        cudaStream_t stream);
int gemm_n_tiles(int N, int block_n);
// ---- stream-K variant for decode (M <= 128): persistent, one CTA per SM; work unit = (n_tile, 64-wide k block),
// units dealt out contiguously so every SM streams the same number of weight bytes.  Each CTA writes the fp32
// partial of every tile segment it owns to ws[slot = cta + tile][128][BN]; consumers (sk_* kernels) add a tile's
// partials in CTA order — a fixed order, so results are run-to-run deterministic — and apply bias / residual /
// RMSNorm / RoPE / SwiGLU while they are at it.
struct StreamK {
    float* ws; int bn, kb, n_tiles, G, rows; long long total;  // rows = 128 or 256 accumulator rows per slot      // kb = k blocks per tile, total = n_tiles * kb, G = CTAs
    int l2_prefetch_units;                                    // weight tiles each CTA prefetches into L2 before griddepcontrol.wait
};
StreamK make_streamk(float* ws, int N, int K, int bn, int G, int rows = 128, bool fp8 = false);   // fp8: 128-wide k blocks
// CTA c owns units [c*total/G, (c+1)*total/G), so unit u lives in CTA floor(((u+1)*G - 1) / total): the CTAs holding the first and the
// last k-block of `tile`.  One definition for the kernels, the consumers and the host plan (32-bit products: host-checked per model).
#ifdef __CUDACC__
__host__ __device__
#endif
inline void sk_tile_ctas(const StreamK& sk, uint32_t tile, uint32_t& c_first, uint32_t& c_last) {
    const uint32_t ut0 = tile * (uint32_t)sk.kb, G = (uint32_t)sk.G, total = (uint32_t)sk.total;
    c_first = ((ut0 + 1u) * G - 1u) / total;
    c_last = ((ut0 + (uint32_t)sk.kb) * G - 1u) / total;
}

size_t streamk_ws_bytes(int N, int bn, int G, int rows = 128);
// every stream-K launcher takes fp8 operands with non-null w8 scales (sk from make_streamk(..., fp8 = true); BN <= 128)
cudaError_t launch_gemm_streamk(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, cudaStream_t stream,
                                W8Scales w8 = {});
// gate/up projection with the SwiGLU finished inside the GEMM (BN=128, one row tile): act[M,F] = silu(gate)*up, bit-identical to
// launch_gemm_streamk + launch_sk_swiglu.  tile_flags: >= n_tiles counters, zero between launches (the kernel re-arms them).
cudaError_t launch_gemm_streamk_swiglu(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int F, int K, const StreamK& sk, void* act,
                                       unsigned int* tile_flags, cudaStream_t stream, W8Scales w8 = {});
// x[T,H] (bf16, in place) += sum of partials; xn = rmsnorm(x) * gain
cudaError_t launch_sk_resid_rmsnorm(const StreamK& sk, void* x, const void* gain, void* xn, int T, int H, float eps, cudaStream_t s);
// act[T,F] = silu(gate) * up from the interleaved gate/up partials (N = 2F)
cudaError_t launch_sk_swiglu(const StreamK& sk, void* act, int T, int F, cudaStream_t s);

struct SkRopeArgs {       // q/k/v from the qkv projection's partials (+ bias): sum -> bf16 -> RoPE -> bf16 (the oracle's order)
    const uint16_t* bias; const int32_t* positions; const int32_t* slots; const float* rope_cos; const float* rope_sin;
    uint16_t* q_out; uint16_t* kv_base; int64_t k_plane_row0, v_plane_row0; int32_t page_size, nh, nkv, D;
    int32_t kv_fp8; float k_inv_scale, v_inv_scale;   // fp8 cache: stored byte = e4m3(value * inv_scale) (KvLayout)
};
// o / down projection with the residual add finished inside the GEMM: x[M, ldx] (bf16, in place) += A.B^T, bit-identical to
// launch_gemm_streamk + the sum/residual half of launch_sk_resid_rmsnorm.  Follow with launch_rmsnorm_wide for the norm.
cudaError_t launch_gemm_streamk_resid(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, void* x, int ldx,
                                      unsigned int* tile_flags, cudaStream_t stream, W8Scales w8 = {});
// qkv projection with bias + RoPE + the paged-KV write finished inside the GEMM (no qkv tensor, no consumer launch), bit-identical to
// launch_gemm_streamk + launch_sk_rope_kv_write
cudaError_t launch_gemm_streamk_rope(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, const SkRopeArgs& rope,
                                     unsigned int* tile_flags, cudaStream_t stream, W8Scales w8 = {});
// ---- cluster split-K GEMM for projections with few output tiles (gemm_clusterk.cu): S CTAs of one cluster own one 128-column tile and 1/S
// of K each, reduce through distributed shared memory and finish the epilogue together (no partial workspace, no consumer launch) ----
int clusterk_pick(int N, int K, int sms, int min_fill_pct = 80);        // cluster size for this shape (8, 4, 3, 2) or 0 = keep the stream-K path
cudaError_t launch_gemm_clusterk_resid(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int S, void* x, int ldx, cudaStream_t stream);
cudaError_t launch_gemm_clusterk_rope(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int S, const SkRopeArgs& rope, cudaStream_t stream);
// xn = rmsnorm(x) * gain with exactly the reduction order of launch_sk_resid_rmsnorm (512 threads per row)
cudaError_t launch_rmsnorm_wide(const void* x, const void* gain, void* xn, int T, int H, float eps, cudaStream_t s);
constexpr int SK_MAX_FLAG_TILES = 1024;      // per-projection capacity of the per-tile piece counters the fused stream-K epilogues use

// reduce EPI_LOGITS partials: out_ids[M] = argmax over n_tiles (ties -> lowest column index)
cudaError_t launch_argmax_reduce(const float* amax_val, const int* amax_idx, int M, int n_tiles, int32_t* out_ids,
                                 float* out_val, cudaStream_t stream);


// ---- elementwise (elementwise.cu) -----------------------------------------------------------
cudaError_t launch_embed_gather(const int32_t* ids, const void* table, void* out, int T, int H, int vocab, cudaStream_t s);
cudaError_t launch_rmsnorm(const void* x, const void* gain, void* y, int T, int H, float eps, cudaStream_t s);
// gather rows: out[i,:] = x[rows[i],:]
cudaError_t launch_gather_rows(const void* x, const int32_t* rows, void* out, int n, int H, cudaStream_t s);
// fp8 (e4m3) rows: x bf16 [R, C] -> q [R, C] bytes + scale [R] fp32, per row s = w8_row_scale(amax) and q = e4m3(x / s) (round to nearest
// even, saturating).  Weights at load time and every projection input of the fp8-weight forward.  C % 16 == 0.
cudaError_t launch_quant_rows_e4m3(const void* x, uint8_t* q, float* scale, int R, int C, cudaStream_t s);
// RoPE (HF rotate_half pairing) on q and k in `qkv` [T, (nh+2nkv)*D]; rotated q -> q_out [T, nh*D];
// rotated k and v -> paged KV cache rows.  slot[t] = page*page_size + offset of token t.
struct KvLayout {
    void* base;            // rows of D elements (bf16, or e4m3 bytes when fp8)
    int64_t layer_stride_rows;   // rows between consecutive layers (= 2 * num_pages * nkv * page_size)
    int64_t kv_stride_rows;      // rows between K and V planes of a layer (= num_pages * nkv * page_size)
    int32_t page_size, n_kv, head_dim, num_pages;
    // fp8 (e4m3) cache: one (page, kv head) block is 64 * D bytes; K as [64 tokens][D], V transposed as [D][64 tokens].  The byte x of
    // layer l decodes to e4m3(x) * k_scale[l] (K) or * v_scale[l] (V); k_scale / v_scale are host arrays of the layers' scales
    int32_t fp8;
    const float* k_scale; const float* v_scale;
};
// same, but q/k/v come from stream-K partials (+ bias): sum -> bf16 round -> RoPE -> bf16 round (the oracle's order)
cudaError_t launch_sk_rope_kv_write(const StreamK& sk, const void* bias, const int32_t* positions, const int32_t* slots,
                                    const float* rope_cos, const float* rope_sin, void* q_out, const KvLayout& kv, int layer, int T,
                                    int nh, cudaStream_t s);
SkRopeArgs make_sk_rope_args(const void* bias, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin,
                             void* q_out, const KvLayout& kv, int layer, int nh);
cudaError_t launch_rope_kv_write(const void* qkv, const int32_t* positions, const int32_t* slots, const float* rope_cos,
                                 const float* rope_sin, void* q_out, const KvLayout& kv, int layer, int T, int nh,
                                 cudaStream_t s);

// ---- weights (weights.cu): deterministic seeded init, bit-identical to oracle gen ----------------
// logical tensor [rows, cols]; `interleave16_with` >= 0 means this is the fused gate/up tensor: physical
// row r holds gate row (r/32)*16+r%16 when (r%32)<16 (tensor_id), else the same row of tensor `tensor_id_b`.
cudaError_t launch_init_weight(void* dst, uint64_t seed, uint64_t tensor_id, int64_t tensor_id_b, int64_t rows, int64_t cols,
                               float std, float mean, cudaStream_t s, int64_t row_off = 0, int64_t col_off = 0, int64_t logical_cols = 0);

// ---- attention (attention.cu) ----------------------------------------------------------------
struct DecodeSeg {        // one contiguous piece of one (sequence, kv head) handled by one CTA
    int32_t seq, kvh, chunk_begin, chunk_end;   // chunks of 64 tokens
    int32_t partial_slot;                        // index into the partial workspace, or -1: single-piece, write final
    int32_t slot_begin, n_pieces, item;          // cut items: first slot, piece count and merge-counter index of the (seq, kv head) item
};
struct DecodeAttnParams {
    const void* q;                 // bf16 [B, nh*D] (already rotated)
    void* out;                     // bf16 [B, nh*D]
    const int32_t* block_tables;   // [B, max_pages_per_seq]
    const int32_t* ctx_lens;       // [B] tokens in cache including the current one
    int32_t max_pages_per_seq;
    const DecodeSeg* segs; const int32_t* cta_seg_ptr; int32_t n_ctas;   // CTA c runs segs[ptr[c] .. ptr[c+1])
    float* part_o; float* part_ml; // partial workspace: [slots, group, D] fp32 and [slots, group, 2]
    int32_t* merge_counters;       // [items], zero at the start of a step; the CTA that completes an item's last piece merges it (null: separate merge kernel)
    int32_t layer, n_heads, n_kv;
    float scale_log2e;             // (1/sqrt(D)) * log2(e)  (the fp8 launcher multiplies in the layer's k_scale)
};
cudaError_t launch_decode_attention(const CUtensorMap* tm_kv, const KvLayout& kv, const DecodeAttnParams& p, cudaStream_t s);
struct MergeItem { int32_t seq, kvh, slot_begin, n_slots; };
cudaError_t launch_decode_merge(const MergeItem* items, int n_items, const float* part_o, const float* part_ml, void* out,
                                int n_heads, int n_kv, int head_dim, cudaStream_t s);

constexpr int PREFILL_TILE_ROWS = 128;                     // query rows of one (tile, head) CTA
struct PrefillTile { int32_t seq, q_row0, pos0, n_rows; };  // <= PREFILL_TILE_ROWS rows of one sequence; q_row0 = row in the token batch
struct PrefillAttnParams {
    const void* q; void* out;      // bf16 [T, nh*D]
    const int32_t* block_tables; int32_t max_pages_per_seq;
    const PrefillTile* tiles; int32_t n_tiles;
    int32_t layer, n_heads, n_kv;
    float scale_log2e;
};
cudaError_t launch_prefill_attention(const CUtensorMap* tm_kv, const KvLayout& kv, const PrefillAttnParams& p, cudaStream_t s);

// bookkeeping for bench.py's gpu_launches claim
uint64_t launches_total();
bool pdl_enabled();     // OA_PDL=0 disables programmatic dependent launch
void count_launch();


// cudaFuncSetAttribute is per device: remember per (kernel instantiation, device) that the dynamic-smem limit has been raised
template <typename K>
inline cudaError_t ensure_dynamic_smem(K kern, int bytes, bool (&done)[16]) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 16 || !done[dev]) {
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 16) done[dev] = true;
    }
    return cudaSuccess;
}

// A launch grid, optionally of thread-block clusters of `cluster` CTAs along x (a dim3 converts to a grid without clusters).
struct LaunchGrid {
    dim3 dim; unsigned cluster;
    LaunchGrid(dim3 d, unsigned cluster_x = 1) : dim(d), cluster(cluster_x) {}
};
// Every kernel launch goes through here: counts it and (unless OA_PDL=0) marks it for programmatic dependent launch.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), LaunchGrid grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid.dim; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    unsigned n = 0;
    if (grid.cluster > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = grid.cluster; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
        ++n;
    }
    if (pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    cfg.attrs = attr; cfg.numAttrs = n;
    count_launch();
    return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

}  // namespace oa
