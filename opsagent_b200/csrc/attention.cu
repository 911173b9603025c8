// attention.cu — paged-KV grouped-query attention for the ReAct decode path.
//
// KV cache (see KvLayout): one bf16 matrix of D-wide rows; row index =
//     ((layer*2 + {0:K,1:V}) * num_pages + page) * n_kv * 64 + kv_head * 64 + token_in_page
// so one (page, kv_head) block is 64 contiguous rows = 64*D*2 bytes, fetched by TMA as D/64 boxes of
// {64 cols, 64 rows} with the 128-byte swizzle (conflict-free ldmatrix reads).
//
// Decode kernel (HBM-bound: every K/V byte is used once, arithmetic intensity ~ group size):
//   warp 4      : TMA producer, streams K and V pages of its (sequence, kv-head) segments through a 3-stage
//                 ring (32 KB/stage for D=128) — bytes in flight per SM = 2 CTAs x 96 KB.
//   warps 0..3  : each owns a 16-token quarter of every 64-token page: S = Q·K^T (mma.sync m16n8k16, the GQA
//                 group's heads in the M rows), online softmax in registers, O += P·V; per-warp (m, l, O)
//                 states are merged once per segment through 12 KB of shared memory.
//   Long or ragged contexts are cut into segments by a host-made plan; partial (m, l, O) go to a workspace and
//   decode_merge_kernel combines them (flash-decoding).
// The 16-row mma.sync tile is the right tool here: with <= 8 real rows per tile even the legacy tensor path
// has far more throughput than the HBM stream it has to keep up with, and a 64-row wgmma tile would be mostly padding.
//
// Prefill kernel: FlashAttention-2 style, 8 warps x 16 query rows per CTA (one TMA-fed K/V stage serves 128 query rows), same TMA ring over the paged cache
// (new tokens' K/V are written to the cache by rope_kv_write before attention), causal mask by position; both products on wgmma.
#include "common.cuh"
#include "kernels.hpp"

namespace oa {

static constexpr int PAGE = 64;             // tokens per page == tokens per pipeline stage
static constexpr int ATT_THREADS = 160;     // 4 consumer warps + 1 producer warp

template <int D>
struct AttCfg {
    static constexpr int HALVES = D / 64;
    static constexpr int TILE_BYTES = PAGE * 128;            // one 64-column half of 64 tokens
    static constexpr int KV_BYTES = HALVES * TILE_BYTES;     // K (or V) of one stage
    static constexpr int STAGE_BYTES = 2 * KV_BYTES;
    static constexpr int STAGES = (D == 128) ? 3 : 4;
    static constexpr int SCRATCH_BYTES = 3 * (D / 4) * 32 * 4;   // 3 warps x (D/8 tiles x 2 regs) x 32 lanes fp32
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + SCRATCH_BYTES + 4 * 8 * 2 * 4 + 2 * STAGES * 8 + 1024;
};

// fp8 cache (KvLayout::fp8): a (page, kv head) block is 64 * D bytes, K as [64 tokens][D] and V as [D][64 tokens].  TMA reads the pool as
// rows of 128 bytes (make_tmap_u8_2d, box {128, D/2}: one block per load) with the 128-byte swizzle, so byte o of a staged block
// sits at fp8_swz(o).  Decode builds its mma operands straight from these bytes; prefill widens each stage to bf16 first.
template <int D, bool FP8>
struct DecCfg {
    static constexpr int KV_BYTES = FP8 ? PAGE * D : AttCfg<D>::KV_BYTES;
    static constexpr int STAGE_BYTES = 2 * KV_BYTES;
    static constexpr int STAGES = FP8 ? 2 * AttCfg<D>::STAGES : AttCfg<D>::STAGES;     // same bytes in flight per SM
    static constexpr int SCRATCH_BYTES = AttCfg<D>::SCRATCH_BYTES;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + SCRATCH_BYTES + 4 * 8 * 2 * 4 + 2 * STAGES * 8 + 1024;
};
OA_DEVINL uint32_t fp8_swz(uint32_t o) { return o ^ (((o >> 7) & 7u) << 4); }
// row of the pool's 128-byte view where the fp8 block starting at token row `row` (KvLayout rows of D elements) begins
template <int D>
OA_DEVINL int32_t fp8_tma_row(int64_t row) { return (int32_t)(row * D / 128); }

// byte offset of the 16-byte chunk holding (row r, columns d..d+7) inside one K or V stage buffer
template <int D>
OA_DEVINL uint32_t kv_off(int r, int d) {
    return (uint32_t)((d >> 6) * AttCfg<D>::TILE_BYTES + r * 128 + ((((d & 63) >> 3) ^ (r & 7)) << 4));
}

OA_DEVINL void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// =============================================================================================
// decode
// =============================================================================================
// FP8: K / V bytes of the fp8 cache.  The token order inside a warp's 16-token quarter is permuted so that both products read their fp8
// operand along its reduction dimension with plain ldmatrix: S column 2t+e of n-tile j is token 4t+2j+e, and the head dims of each
// 16-wide k-step are paired (4t, 4t+1) / (4t+2, 4t+3) in Q and K alike.  P's fragment then holds tokens 4t..4t+3, which is what an
// ldmatrix row of the transposed V block gives.  k_scale is in p.scale_log2e; v_scale multiplies the output.
template <int D, bool FP8>
__global__ void __launch_bounds__(ATT_THREADS, 2) decode_attention_kernel(const __grid_constant__ CUtensorMap tm_kv,
                                                                          const DecodeAttnParams p, const int64_t layer_row0,
                                                                          const int64_t kv_stride_rows, const float v_scale) {
    using Cfg = DecCfg<D, FP8>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int KS = D / 16;      // k-steps of Q·K^T
    constexpr int NT = D / 8;       // n-tiles of P·V
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* scratch = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
    float* ml_s = scratch + Cfg::SCRATCH_BYTES / 4;          // [4 warps][8 rows][2]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(ml_s + 64);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = p.n_heads / p.n_kv;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_kv);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch();

    // plan, block tables and context lengths were copied in before the first kernel of the step: safe to read now
    const int seg_begin = p.cta_seg_ptr[blockIdx.x], seg_end = p.cta_seg_ptr[blockIdx.x + 1];

    if (warp == 4) {
        // ------------------------------- producer -------------------------------
        // Pages strictly before the one holding this step's token are immutable, so their K/V stream may start
        // before the predecessor (RoPE + KV-page write) has finished; wait lazily, at the first page that may change
        // or once the ring is full.
        if (lane == 0) {
            int s = 0; uint32_t ph = 0; int issued = 0; bool waited = false;
            for (int si = seg_begin; si < seg_end; ++si) {
                const DecodeSeg sg = p.segs[si];
                const int32_t* bt = p.block_tables + (size_t)sg.seq * p.max_pages_per_seq;
                const int mutable_chunk = (p.ctx_lens[sg.seq] - 1) / PAGE;
                for (int c = sg.chunk_begin; c < sg.chunk_end; ++c) {
                    if (!waited && (issued >= STAGES || c >= mutable_chunk)) { griddep_wait(); waited = true; }
                    ++issued;
                    const int page = bt[c];
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* kdst = smem + s * Cfg::STAGE_BYTES;
                    uint8_t* vdst = kdst + Cfg::KV_BYTES;
                    mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
                    const int64_t krow = layer_row0 + ((int64_t)page * p.n_kv + sg.kvh) * PAGE;
                    const int64_t vrow = krow + kv_stride_rows;
                    if constexpr (FP8) {
                        tma_load_2d(kdst, &tm_kv, &full_bar[s], 0, fp8_tma_row<D>(krow), kEvictFirst);
                        tma_load_2d(vdst, &tm_kv, &full_bar[s], 0, fp8_tma_row<D>(vrow), kEvictFirst);
                    } else {
#pragma unroll
                        for (int h = 0; h < AttCfg<D>::HALVES; ++h) {
                            tma_load_2d(kdst + h * AttCfg<D>::TILE_BYTES, &tm_kv, &full_bar[s], h * 64, (int32_t)krow, kEvictFirst);
                            tma_load_2d(vdst + h * AttCfg<D>::TILE_BYTES, &tm_kv, &full_bar[s], h * 64, (int32_t)vrow, kEvictFirst);
                        }
                    }
                    if (++s == STAGES) { s = 0; ph ^= 1; }
                }
            }
        }
        return;
    }

    // ------------------------------- consumers -------------------------------
    griddep_wait();       // Q comes from the predecessor; partial/out buffers may still be read by it
    const int g = lane >> 2, t = lane & 3;
    int s = 0; uint32_t ph = 0;
    for (int si = seg_begin; si < seg_end; ++si) {
        const DecodeSeg sg = p.segs[si];
        const int ctx = p.ctx_lens[sg.seq];
        // Q fragments: rows = heads of this kv group (rows >= grp are zero)
        uint32_t qa[KS][2];
        {
            const uint16_t* qrow = reinterpret_cast<const uint16_t*>(p.q) + (size_t)sg.seq * p.n_heads * D + (size_t)(sg.kvh * grp + g) * D;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
                if (g < grp) {
                    const int d0 = FP8 ? 4 * t : 2 * t, d1 = FP8 ? 4 * t + 2 : 8 + 2 * t;
                    qa[ks][0] = *reinterpret_cast<const uint32_t*>(qrow + ks * 16 + d0);
                    qa[ks][1] = *reinterpret_cast<const uint32_t*>(qrow + ks * 16 + d1);
                } else { qa[ks][0] = 0u; qa[ks][1] = 0u; }
            }
        }
        float oacc[NT][4];
#pragma unroll
        for (int j = 0; j < NT; ++j) { oacc[j][0] = oacc[j][1] = oacc[j][2] = oacc[j][3] = 0.f; }
        float m_run = -INFINITY, l_run = 0.f;

        for (int c = sg.chunk_begin; c < sg.chunk_end; ++c) {
            mbar_wait(&full_bar[s], ph);
            const int tok0 = c * PAGE + warp * 16;        // first token of this warp's quarter
            if (tok0 < ctx) {
                const uint32_t kbase = smem_u32(smem + s * Cfg::STAGE_BYTES);
                const uint32_t vbase = kbase + Cfg::KV_BYTES;
                float sacc[2][4];
#pragma unroll
                for (int j = 0; j < 2; ++j) { sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f; }
                if constexpr (FP8) {
                    // matrix m = lane / 8 of each ldmatrix.x4: n-tile m & 1, k-step 2kk + (m >> 1); its row c = lane % 8 is token 4(c/2) + 2(m&1) + c%2
                    const int m = lane >> 3, c = lane & 7;
                    const uint32_t row0 = (uint32_t)(warp * 16 + 4 * (c >> 1) + 2 * (m & 1) + (c & 1)) * D + (uint32_t)(m >> 1) * 16;
#pragma unroll
                    for (int kk = 0; kk < KS / 2; ++kk) {
                        uint32_t r[4];
                        ldmatrix_x4(kbase + fp8_swz(row0 + kk * 32), r[0], r[1], r[2], r[3]);
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int ks = 2 * kk + (i >> 1);
                            mma_bf16_16816(sacc[i & 1], qa[ks][0], 0u, qa[ks][1], 0u, e4m3x2_to_bf16x2((uint16_t)r[i]), e4m3x2_to_bf16x2((uint16_t)(r[i] >> 16)));
                        }
                    }
                } else {
                    const int r = warp * 16 + ((lane >> 4) << 3) + (lane & 7);
                    const int dsel = ((lane >> 3) & 1) << 3;
#pragma unroll
                    for (int ks = 0; ks < KS; ++ks) {
                        uint32_t b0, b1, b2, b3;
                        ldmatrix_x4(kbase + kv_off<D>(r, ks * 16 + dsel), b0, b1, b2, b3);
                        mma_bf16_16816(sacc[0], qa[ks][0], 0u, qa[ks][1], 0u, b0, b1);
                        mma_bf16_16816(sacc[1], qa[ks][0], 0u, qa[ks][1], 0u, b2, b3);
                    }
                }
                // scaled scores (log2 domain) + tail mask; row g lives in sacc[j][0..1]
                float sc[4];
#pragma unroll
                for (int j = 0; j < 2; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int tok = tok0 + (FP8 ? 4 * t + 2 * j : j * 8 + 2 * t) + e;
                        sc[j * 2 + e] = tok < ctx ? sacc[j][e] * p.scale_log2e : -INFINITY;
                    }
                float mx = fmaxf(fmaxf(sc[0], sc[1]), fmaxf(sc[2], sc[3]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_new = fmaxf(m_run, mx);              // finite: the quarter has >= 1 valid token
                const float alpha = exp2f(m_run - m_new);
                float pr[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) pr[e] = exp2f(sc[e] - m_new);
                l_run = l_run * alpha + (pr[0] + pr[1] + pr[2] + pr[3]);
                m_run = m_new;
                const uint32_t pa0 = pack_bf16x2(pr[0], pr[1]), pa2 = pack_bf16x2(pr[2], pr[3]);
                if constexpr (FP8) {
                    // matrix m of ldmatrix.x4 number jj: n-tile 4jj + m, rows = its 8 head dims, 16 bytes = this warp's 16 tokens
                    const uint32_t row0 = (uint32_t)(8 * (lane >> 3) + (lane & 7)) * PAGE + warp * 16;
#pragma unroll
                    for (int j = 0; j < NT; ++j) { oacc[j][0] *= alpha; oacc[j][1] *= alpha; }
#pragma unroll
                    for (int jj = 0; jj < NT / 4; ++jj) {
                        uint32_t r[4];
                        ldmatrix_x4(vbase + fp8_swz(row0 + jj * 32 * PAGE), r[0], r[1], r[2], r[3]);
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            mma_bf16_16816(oacc[4 * jj + i], pa0, 0u, pa2, 0u, e4m3x2_to_bf16x2((uint16_t)r[i]), e4m3x2_to_bf16x2((uint16_t)(r[i] >> 16)));
                    }
                } else {
                    const int r = warp * 16 + (((lane >> 3) & 1) << 3) + (lane & 7);
                    const int dsel = (lane >> 4) << 3;
#pragma unroll
                    for (int j = 0; j < NT; j += 2) {
                        uint32_t b0, b1, b2, b3;
                        ldmatrix_x4_trans(vbase + kv_off<D>(r, j * 8 + dsel), b0, b1, b2, b3);
                        oacc[j][0] *= alpha; oacc[j][1] *= alpha; oacc[j + 1][0] *= alpha; oacc[j + 1][1] *= alpha;
                        mma_bf16_16816(oacc[j], pa0, 0u, pa2, 0u, b0, b1);
                        mma_bf16_16816(oacc[j + 1], pa0, 0u, pa2, 0u, b2, b3);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[s]);
            if (++s == STAGES) { s = 0; ph ^= 1; }
        }

        // ---- merge the four warps' states (warp 0 accumulates) ----
        l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
        l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
        if (t == 0) { ml_s[(warp * 8 + g) * 2] = m_run; ml_s[(warp * 8 + g) * 2 + 1] = l_run; }
        if (warp > 0) {
            float* dst = scratch + (size_t)(warp - 1) * (NT * 2) * 32;
#pragma unroll
            for (int j = 0; j < NT; ++j) { dst[(j * 2) * 32 + lane] = oacc[j][0]; dst[(j * 2 + 1) * 32 + lane] = oacc[j][1]; }
        }
        named_bar_sync(1, 128);
        if (warp == 0) {
            float mw[4], lw[4];
#pragma unroll
            for (int w = 0; w < 4; ++w) { mw[w] = ml_s[(w * 8 + g) * 2]; lw[w] = ml_s[(w * 8 + g) * 2 + 1]; }
            const float m_tot = fmaxf(fmaxf(mw[0], mw[1]), fmaxf(mw[2], mw[3]));
            float f[4], l_tot = 0.f;
#pragma unroll
            for (int w = 0; w < 4; ++w) { f[w] = exp2f(mw[w] - m_tot); l_tot += f[w] * lw[w]; }
#pragma unroll
            for (int j = 0; j < NT; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float o = oacc[j][e] * f[0];
#pragma unroll
                    for (int w = 1; w < 4; ++w) o += f[w] * scratch[(size_t)(w - 1) * (NT * 2) * 32 + (j * 2 + e) * 32 + lane];
                    oacc[j][e] = o;
                }
            if (g < grp) {
                if (sg.partial_slot < 0) {
                    const float inv = (FP8 ? v_scale : 1.0f) / l_tot;
                    uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (size_t)sg.seq * p.n_heads * D + (size_t)(sg.kvh * grp + g) * D;
#pragma unroll
                    for (int j = 0; j < NT; ++j)
                        *reinterpret_cast<uint32_t*>(orow + j * 8 + 2 * t) = pack_bf16x2(oacc[j][0] * inv, oacc[j][1] * inv);
                } else {
                    float* po = p.part_o + ((size_t)sg.partial_slot * grp + g) * D;
#pragma unroll
                    for (int j = 0; j < NT; ++j) {
                        if constexpr (FP8) *reinterpret_cast<float2*>(po + j * 8 + 2 * t) = make_float2(oacc[j][0] * v_scale, oacc[j][1] * v_scale);
                        else *reinterpret_cast<float2*>(po + j * 8 + 2 * t) = make_float2(oacc[j][0], oacc[j][1]);
                    }
                    if (t == 0) {
                        p.part_ml[((size_t)sg.partial_slot * grp + g) * 2] = m_tot;
                        p.part_ml[((size_t)sg.partial_slot * grp + g) * 2 + 1] = l_tot;
                    }
                }
            }
            if (sg.partial_slot >= 0 && p.merge_counters) {
                // flash-decoding merge without a second kernel: the CTA that finishes an item's LAST piece combines all pieces.
                // Counters advance by n_pieces per layer and start each step at zero, so "last" is a multiple of n_pieces.
                __threadfence();
                __syncwarp();
                int last = 0;
                if (lane == 0) last = ((atomicAdd(p.merge_counters + sg.item, 1) + 1) % sg.n_pieces) == 0;
                last = __shfl_sync(0xffffffffu, last, 0);
                if (last) {
                    __threadfence();
                    if (g < grp) {
                        float m_all = -INFINITY;
                        for (int i = 0; i < sg.n_pieces; ++i) m_all = fmaxf(m_all, __ldcg(p.part_ml + ((size_t)(sg.slot_begin + i) * grp + g) * 2));
                        float l_all = 0.f;
#pragma unroll
                        for (int j = 0; j < NT; ++j) { oacc[j][0] = 0.f; oacc[j][1] = 0.f; }
                        for (int i = 0; i < sg.n_pieces; ++i) {                       // slot order: deterministic
                            const size_t sl = (size_t)(sg.slot_begin + i) * grp + g;
                            const float f = exp2f(__ldcg(p.part_ml + sl * 2) - m_all);
                            l_all += f * __ldcg(p.part_ml + sl * 2 + 1);
                            const float* pi = p.part_o + sl * D;
#pragma unroll
                            for (int j = 0; j < NT; ++j) { const float2 v2 = __ldcg(reinterpret_cast<const float2*>(pi + j * 8 + 2 * t)); oacc[j][0] += f * v2.x; oacc[j][1] += f * v2.y; }
                        }
                        const float inv = 1.0f / l_all;
                        uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (size_t)sg.seq * p.n_heads * D + (size_t)(sg.kvh * grp + g) * D;
#pragma unroll
                        for (int j = 0; j < NT; ++j)
                            *reinterpret_cast<uint32_t*>(orow + j * 8 + 2 * t) = pack_bf16x2(oacc[j][0] * inv, oacc[j][1] * inv);
                    }
                }
            }
        }
        named_bar_sync(1, 128);   // scratch free for the next segment
    }
}

// out[seq, head, :] = sum_i 2^(m_i - m) o_i / sum_i 2^(m_i - m) l_i over the item's partial slots
__global__ void decode_merge_kernel(const MergeItem* __restrict__ items, const float* __restrict__ part_o,
                                    const float* __restrict__ part_ml, uint16_t* __restrict__ out, int n_heads, int n_kv, int D) {
    griddep_launch(); griddep_wait();
    const MergeItem it = items[blockIdx.x];
    const int grp = n_heads / n_kv;
    for (int idx = threadIdx.x; idx < grp * D; idx += blockDim.x) {
        const int g = idx / D, d = idx - g * D;
        float m_tot = -INFINITY;
        for (int i = 0; i < it.n_slots; ++i) m_tot = fmaxf(m_tot, part_ml[((size_t)(it.slot_begin + i) * grp + g) * 2]);
        float o = 0.f, l = 0.f;
        for (int i = 0; i < it.n_slots; ++i) {
            const size_t sl = (size_t)(it.slot_begin + i) * grp + g;
            const float f = exp2f(part_ml[sl * 2] - m_tot);
            o += f * part_o[sl * D + d];
            l += f * part_ml[sl * 2 + 1];
        }
        out[(size_t)it.seq * n_heads * D + (size_t)(it.kvh * grp + g) * D + d] = f32_to_bf16_bits(o / l);
    }
}

cudaError_t launch_decode_merge(const MergeItem* items, int n_items, const float* part_o, const float* part_ml, void* out,
                                int n_heads, int n_kv, int head_dim, cudaStream_t s) {
    if (n_items <= 0) return cudaSuccess;
    return launch_k(decode_merge_kernel, dim3(n_items), dim3(128), 0, s, items, part_o, part_ml, reinterpret_cast<uint16_t*>(out), n_heads, n_kv, head_dim);
}

template <int D, bool FP8>
static cudaError_t launch_decode_d(const CUtensorMap* tm_kv, const KvLayout& kv, const DecodeAttnParams& p, cudaStream_t s) {
    auto kern = decode_attention_kernel<D, FP8>;
    constexpr int SMEM = DecCfg<D, FP8>::SMEM_BYTES;
    static bool attr_done[16] = {};
    { cudaError_t e = ensure_dynamic_smem(kern, SMEM, attr_done); if (e != cudaSuccess) return e; }
    DecodeAttnParams q = p;
    float v_scale = 1.0f;
    if (FP8) { q.scale_log2e = p.scale_log2e * kv.k_scale[p.layer]; v_scale = kv.v_scale[p.layer]; }
    return launch_k(kern, dim3(p.n_ctas), dim3(ATT_THREADS), SMEM, s, *tm_kv, q, (int64_t)p.layer * kv.layer_stride_rows, kv.kv_stride_rows, v_scale);
}

cudaError_t launch_decode_attention(const CUtensorMap* tm_kv, const KvLayout& kv, const DecodeAttnParams& p, cudaStream_t s) {
    if (p.n_ctas <= 0) return cudaSuccess;
    if (kv.page_size != PAGE || p.n_heads % p.n_kv != 0 || p.n_heads / p.n_kv > 8) return cudaErrorInvalidValue;
    if (kv.head_dim == 128) return kv.fp8 ? launch_decode_d<128, true>(tm_kv, kv, p, s) : launch_decode_d<128, false>(tm_kv, kv, p, s);
    if (kv.head_dim == 64) return kv.fp8 ? launch_decode_d<64, true>(tm_kv, kv, p, s) : launch_decode_d<64, false>(tm_kv, kv, p, s);
    return cudaErrorInvalidValue;
}

// =============================================================================================
// prefill (causal, paged)
// =============================================================================================
static constexpr int PREFILL_WARPS = PREFILL_TILE_ROWS / 16;            // 8 consumer warps x 16 query rows share every K/V stage
static constexpr int PREFILL_THREADS = (PREFILL_WARPS + 1) * 32;        // + 1 TMA producer warp

template <int D, bool FP8>
struct PreCfg {
    static constexpr int RING_BYTES = FP8 ? 2 * PAGE * D : AttCfg<D>::STAGE_BYTES;        // one TMA stage (K and V of one page)
    static constexpr int STAGES = FP8 ? 4 : AttCfg<D>::STAGES;
    static constexpr int WIDE_BYTES = FP8 ? 2 * AttCfg<D>::STAGE_BYTES : 0;               // fp8: two bf16 copies of a stage (double buffer)
    static constexpr int SMEM_BYTES = STAGES * RING_BYTES + WIDE_BYTES + 2 * STAGES * 8 + 1024;
};

// fp8 prefill: the consumer warps widen a staged page to bf16 before the wgmma products read it.  K [64][D] bytes -> the bf16 K tile layout
// (kv_off); V [D][64] bytes -> D rows of 64 bf16 tokens with the 128-byte swizzle, i.e. a K-major B operand of P·V.
template <int D>
OA_DEVINL void widen_fp8_stage(const uint8_t* src, uint8_t* dst, int tid) {
    constexpr int CHUNKS = PAGE * D / 16;          // 16-byte chunks of K (and of V)
    auto widen16 = [](uint4 b, uint4& lo, uint4& hi) {
        lo.x = e4m3x2_to_bf16x2((uint16_t)b.x); lo.y = e4m3x2_to_bf16x2((uint16_t)(b.x >> 16));
        lo.z = e4m3x2_to_bf16x2((uint16_t)b.y); lo.w = e4m3x2_to_bf16x2((uint16_t)(b.y >> 16));
        hi.x = e4m3x2_to_bf16x2((uint16_t)b.z); hi.y = e4m3x2_to_bf16x2((uint16_t)(b.z >> 16));
        hi.z = e4m3x2_to_bf16x2((uint16_t)b.w); hi.w = e4m3x2_to_bf16x2((uint16_t)(b.w >> 16));
    };
#pragma unroll
    for (int q = tid; q < CHUNKS; q += PREFILL_WARPS * 32) {
        const int r = q / (D / 16), d0 = (q % (D / 16)) * 16;
        uint4 lo, hi;
        widen16(*reinterpret_cast<const uint4*>(src + fp8_swz((uint32_t)(r * D + d0))), lo, hi);
        *reinterpret_cast<uint4*>(dst + kv_off<D>(r, d0)) = lo;
        *reinterpret_cast<uint4*>(dst + kv_off<D>(r, d0 + 8)) = hi;
    }
#pragma unroll
    for (int q = tid; q < CHUNKS; q += PREFILL_WARPS * 32) {
        const int d = q >> 2, c0 = (q & 3) * 2;        // head dim d, tokens 8 c0 .. 8 c0 + 15
        uint4 lo, hi;
        widen16(*reinterpret_cast<const uint4*>(src + PAGE * D + fp8_swz((uint32_t)(d * PAGE + c0 * 8))), lo, hi);
        uint8_t* row = dst + AttCfg<D>::KV_BYTES + d * 128;
        *reinterpret_cast<uint4*>(row + ((c0 ^ (d & 7)) << 4)) = lo;
        *reinterpret_cast<uint4*>(row + (((c0 + 1) ^ (d & 7)) << 4)) = hi;
    }
}

// Both products on wgmma: warpgroup g (warps 4g..4g+3) owns query rows [64g, 64g + 64).  S = Q·Kᵀ is m64n64k16 with Q from registers (the mma.sync A-fragment layout) and K K-major as TMA stored it;
// O += P·V is m64nDk16 with P from registers and V read MN-major (d contiguous, as stored).  The accumulator fragments have the
// mma.sync C layout (register 4j + e = rows g / g+8, columns 8j + 2t + e), so the online softmax works on them directly.
// FP8: pages of the fp8 cache, widened to bf16 per stage (widen_fp8_stage); V is then K-major.  k_scale is in p.scale_log2e.
template <int D, bool FP8>
__global__ void __launch_bounds__(PREFILL_THREADS, 1) prefill_attention_kernel(const __grid_constant__ CUtensorMap tm_kv,
                                                                           const PrefillAttnParams p, const int64_t layer_row0,
                                                                           const int64_t kv_stride_rows, const float v_scale) {
    using Cfg = AttCfg<D>;
    using PC = PreCfg<D, FP8>;
    constexpr int STAGES = PC::STAGES;
    constexpr int KS = D / 16, NT = D / 8;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* wide = smem + STAGES * PC::RING_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(wide + PC::WIDE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const PrefillTile tile = p.tiles[blockIdx.x];
    const int head = blockIdx.y;
    const int grp = p.n_heads / p.n_kv, kvh = head / grp;
    const int n_chunks = (tile.pos0 + tile.n_rows - 1) / PAGE + 1;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_kv);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], PREFILL_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch();
    griddep_wait();

    if (warp == PREFILL_WARPS) {
        if (lane == 0) {
            const int32_t* bt = p.block_tables + (size_t)tile.seq * p.max_pages_per_seq;
            int s = 0; uint32_t ph = 0;
            for (int c = 0; c < n_chunks; ++c) {
                const int page = bt[c];
                mbar_wait(&empty_bar[s], ph ^ 1);
                uint8_t* kdst = smem + s * PC::RING_BYTES;
                uint8_t* vdst = kdst + PC::RING_BYTES / 2;
                mbar_expect_tx(&full_bar[s], PC::RING_BYTES);
                const int64_t krow = layer_row0 + ((int64_t)page * p.n_kv + kvh) * PAGE;
                const int64_t vrow = krow + kv_stride_rows;
                if constexpr (FP8) {
                    tma_load_2d(kdst, &tm_kv, &full_bar[s], 0, fp8_tma_row<D>(krow), kEvictLast);
                    tma_load_2d(vdst, &tm_kv, &full_bar[s], 0, fp8_tma_row<D>(vrow), kEvictLast);
                } else {
#pragma unroll
                    for (int h = 0; h < Cfg::HALVES; ++h) {
                        tma_load_2d(kdst + h * Cfg::TILE_BYTES, &tm_kv, &full_bar[s], h * 64, (int32_t)krow, kEvictLast);
                        tma_load_2d(vdst + h * Cfg::TILE_BYTES, &tm_kv, &full_bar[s], h * 64, (int32_t)vrow, kEvictLast);
                    }
                }
                if (++s == STAGES) { s = 0; ph ^= 1; }
            }
        }
        return;
    }

    const int g = lane >> 2, t = lane & 3;
    const int r0 = warp * 16 + g, r1 = r0 + 8;                  // this thread's two query rows in the tile
    const int qpos0 = tile.pos0 + r0, qpos1 = tile.pos0 + r1;
    uint32_t qa[KS][4];
    {
        const uint16_t* qb = reinterpret_cast<const uint16_t*>(p.q) + (size_t)head * D;
        const size_t ldq = (size_t)p.n_heads * D;
        const bool ok0 = r0 < tile.n_rows, ok1 = r1 < tile.n_rows;
        const uint16_t* q0 = qb + (size_t)(tile.q_row0 + r0) * ldq;
        const uint16_t* q1 = qb + (size_t)(tile.q_row0 + r1) * ldq;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            qa[ks][0] = ok0 ? *reinterpret_cast<const uint32_t*>(q0 + ks * 16 + 2 * t) : 0u;
            qa[ks][1] = ok1 ? *reinterpret_cast<const uint32_t*>(q1 + ks * 16 + 2 * t) : 0u;
            qa[ks][2] = ok0 ? *reinterpret_cast<const uint32_t*>(q0 + ks * 16 + 8 + 2 * t) : 0u;
            qa[ks][3] = ok1 ? *reinterpret_cast<const uint32_t*>(q1 + ks * 16 + 8 + 2 * t) : 0u;
        }
    }
    float oacc[NT * 4];
#pragma unroll
    for (int i = 0; i < NT * 4; ++i) oacc[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    const int wg_last_pos = tile.pos0 + (warp >> 2) * 64 + 63;   // largest query position of this warpgroup: wgmma is warpgroup-wide

    int s = 0; uint32_t ph = 0;
    for (int c = 0; c < n_chunks; ++c) {
        mbar_wait(&full_bar[s], ph);
        uint32_t kbase = smem_u32(smem + s * Cfg::STAGE_BYTES);
        if constexpr (FP8) {
            // every consumer warp widens its share; the buffer written here was last read for chunk c - 2, which all warps finished
            // before the barrier of chunk c - 1
            uint8_t* w = wide + (c & 1) * Cfg::STAGE_BYTES;
            widen_fp8_stage<D>(smem + s * PC::RING_BYTES, w, threadIdx.x);
            fence_proxy_async();                    // generic-proxy stores -> wgmma operand reads
            named_bar_sync(1, PREFILL_WARPS * 32);
            if (lane == 0) mbar_arrive(&empty_bar[s]);     // every warp has widened its share: the fp8 stage is free for the producer
            kbase = smem_u32(w);
        }
        if (c * PAGE <= wg_last_pos) {
            const uint32_t vbase = kbase + Cfg::KV_BYTES;
            float sacc[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) sacc[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < KS; ++ks)        // 16 head dims per step: +32 B inside the 128-byte row, next 64-column half at +TILE_BYTES
                wgmma_rs_m64n64(sacc, qa[ks], gmma_desc_sw128(kbase + (uint32_t)((ks >> 2) * Cfg::TILE_BYTES + (ks & 3) * 32)), ks > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            const bool diag = (c * PAGE + PAGE - 1) > tile.pos0 + warp * 16;   // some (row, col) pairs may be masked
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int kpos = c * PAGE + j * 8 + 2 * t + e;
                    float v0 = sacc[4 * j + e] * p.scale_log2e, v1 = sacc[4 * j + 2 + e] * p.scale_log2e;
                    if (diag) { if (kpos > qpos0) v0 = -INFINITY; if (kpos > qpos1) v1 = -INFINITY; }
                    sacc[4 * j + e] = v0; sacc[4 * j + 2 + e] = v1;
                    mx0 = fmaxf(mx0, v0); mx1 = fmaxf(mx1, v1);
                }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            // chunk 0 always has key 0 <= every query position, so the running max is finite from the first chunk on; a chunk wholly
            // in a row's future gives mx = -inf and leaves m, l and O unchanged
            const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
            const float al0 = exp2f(m0 - mn0), al1 = exp2f(m1 - mn1);
            m0 = mn0; m1 = mn1;
            float ps0 = 0.f, ps1 = 0.f;
            uint32_t pa[8][2];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float p00 = exp2f(sacc[4 * j] - mn0), p01 = exp2f(sacc[4 * j + 1] - mn0);
                const float p10 = exp2f(sacc[4 * j + 2] - mn1), p11 = exp2f(sacc[4 * j + 3] - mn1);
                ps0 += p00 + p01; ps1 += p10 + p11;
                pa[j][0] = pack_bf16x2(p00, p01); pa[j][1] = pack_bf16x2(p10, p11);
            }
            l0 = l0 * al0 + ps0; l1 = l1 * al1 + ps1;
#pragma unroll
            for (int j = 0; j < NT; ++j) { oacc[4 * j] *= al0; oacc[4 * j + 1] *= al0; oacc[4 * j + 2] *= al1; oacc[4 * j + 3] *= al1; }
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {       // 16 key tokens per step = two 8-row groups of V (1024 B apart)
                const uint32_t a[4] = {pa[2 * kk][0], pa[2 * kk][1], pa[2 * kk + 1][0], pa[2 * kk + 1][1]};
                if constexpr (FP8) {                // widened V: D rows of 64 tokens, K-major (+32 B per 16 tokens)
                    const uint64_t db = gmma_desc_sw128(vbase + (uint32_t)(kk * 32));
                    if constexpr (D == 128) wgmma_rs_m64n128(oacc, a, db, 1u);
                    else wgmma_rs_m64n64(oacc, a, db, 1u);
                } else {
                    const uint64_t db = gmma_desc_sw128_mn(vbase + (uint32_t)(kk * 2048), (uint32_t)Cfg::TILE_BYTES, 1024u);
                    if constexpr (D == 128) wgmma_rs_m64n128_tb(oacc, a, db, 1u);
                    else wgmma_rs_m64n64_tb(oacc, a, db, 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();                        // V of this stage has been read
        }
        __syncwarp();
        if (!FP8 && lane == 0) mbar_arrive(&empty_bar[s]);
        if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = (FP8 ? v_scale : 1.0f) / l0, inv1 = (FP8 ? v_scale : 1.0f) / l1;
    uint16_t* ob = reinterpret_cast<uint16_t*>(p.out) + (size_t)head * D;
    const size_t ldo = (size_t)p.n_heads * D;
    if (r0 < tile.n_rows) {
        uint16_t* o = ob + (size_t)(tile.q_row0 + r0) * ldo;
#pragma unroll
        for (int j = 0; j < NT; ++j) *reinterpret_cast<uint32_t*>(o + j * 8 + 2 * t) = pack_bf16x2(oacc[4 * j] * inv0, oacc[4 * j + 1] * inv0);
    }
    if (r1 < tile.n_rows) {
        uint16_t* o = ob + (size_t)(tile.q_row0 + r1) * ldo;
#pragma unroll
        for (int j = 0; j < NT; ++j) *reinterpret_cast<uint32_t*>(o + j * 8 + 2 * t) = pack_bf16x2(oacc[4 * j + 2] * inv1, oacc[4 * j + 3] * inv1);
    }
}

template <int D, bool FP8>
static cudaError_t launch_prefill_d(const CUtensorMap* tm_kv, const KvLayout& kv, const PrefillAttnParams& p, cudaStream_t s) {
    auto kern = prefill_attention_kernel<D, FP8>;
    constexpr int SMEM = PreCfg<D, FP8>::SMEM_BYTES;
    static bool attr_done[16] = {};
    { cudaError_t e = ensure_dynamic_smem(kern, SMEM, attr_done); if (e != cudaSuccess) return e; }
    dim3 grid(p.n_tiles, p.n_heads, 1);
    PrefillAttnParams q = p;
    float v_scale = 1.0f;
    if (FP8) { q.scale_log2e = p.scale_log2e * kv.k_scale[p.layer]; v_scale = kv.v_scale[p.layer]; }
    return launch_k(kern, grid, dim3(PREFILL_THREADS), SMEM, s, *tm_kv, q, (int64_t)p.layer * kv.layer_stride_rows, kv.kv_stride_rows, v_scale);
}

cudaError_t launch_prefill_attention(const CUtensorMap* tm_kv, const KvLayout& kv, const PrefillAttnParams& p, cudaStream_t s) {
    if (p.n_tiles <= 0) return cudaSuccess;
    if (kv.page_size != PAGE || p.n_heads % p.n_kv != 0) return cudaErrorInvalidValue;
    if (kv.head_dim == 128) return kv.fp8 ? launch_prefill_d<128, true>(tm_kv, kv, p, s) : launch_prefill_d<128, false>(tm_kv, kv, p, s);
    if (kv.head_dim == 64) return kv.fp8 ? launch_prefill_d<64, true>(tm_kv, kv, p, s) : launch_prefill_d<64, false>(tm_kv, kv, p, s);
    return cudaErrorInvalidValue;
}

}  // namespace oa
