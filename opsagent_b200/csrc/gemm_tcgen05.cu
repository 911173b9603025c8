// gemm_tcgen05.cu — C[M,N] = A[M,K] · B[N,K]^T for the QKV / O / gate-up / down / LM-head projections (the file keeps its
// name from the Blackwell version; everything in it is Hopper wgmma).
//
// sm_90a design (one CTA = one 128 x BLOCK_N output tile):
//   warp 8    : TMA producer — cp.async.bulk.tensor 2D boxes {64 x 128} of A and {64 x BLOCK_N} of B into a
//               STAGES-deep shared-memory ring (128-byte swizzle), completion on `full` mbarriers.
//   warps 0-7 : two consumer warpgroups; warpgroup g issues wgmma 64 x BLOCK_N x 16 (bf16 -> fp32 in registers) for rows
//               [64g, 64g + 64) of the tile, releases ring slots (`empty`) as their MMAs retire, and at the end of a tile
//               writes the accumulator into a swizzled fp32 tile in shared memory (`acc_full`).
//   epilogue  : then warpgroup 0, one output row per thread (bias | residual add | SwiGLU | fp32 logits + row arg-max).
// Decode (M <= 128) is weight-streaming and HBM-bound: B tiles are fetched with an evict-first L2 policy, the
// small A operand with evict-last.  K tails and M/N tails rely on TMA zero fill + predicated stores.
//
// The role of this file in the reference's terms: it is the arithmetic that sits behind
// llms.OpenAIClient.Chat (reference pkg/llms/openai.go:69-104) once the `local-cuda` provider replaces the
// remote HTTP server — see DESIGN.md §Kernels.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "kernels.hpp"
#include "sk_consumers.cuh"

namespace oa {

static constexpr int BLOCK_M = 128;
static constexpr int BLOCK_K = 64;     // 64 bf16 = 128 B = one swizzle row
static constexpr int EPI_WARP0 = 0, PRODUCER_WARP = 8;
// 2 consumer warpgroups + 1 producer warp: 9 warps leave 168 registers per thread, room for a 64 x 256 fp32 fragment (128)
static constexpr int GEMM_THREADS = 32 * (PRODUCER_WARP + 1);
#define OA_GEMM_REGS __launch_bounds__(GEMM_THREADS, 1)
static constexpr int RASTER_GROUP_M = 16;
static constexpr int SMEM_LIMIT = 232448;                           // opt-in shared memory of one CTA on sm_90

// Consumer side of the ring: n_kb k-blocks into this warpgroup's registers (rows [64g, 64g + 64) of each of the MT 128-row A tiles).
// One wgmma group stays in flight; a slot is released (one arrival per consumer warp) once the group that read it has retired.
template <int BN, int MT, int STAGES, int STAGE_BYTES, int A_TILE_BYTES, int A_BYTES>
OA_DEVINL void wg_mma_run(float (&d)[MT][BN / 2], uint8_t* smem, uint64_t* full_bar, int& s, uint32_t& ph, int n_kb) {
    uint64_t* empty_bar = full_bar + STAGES;
    const uint32_t g_off = (threadIdx.x >> 7) * 64 * 128;
    const bool leader = (threadIdx.x & 31) == 0;
    int prev = -1;
    for (int i = 0; i < n_kb; ++i) {
        mbar_wait(&full_bar[s], ph);
        const uint32_t st = smem_u32(smem) + (uint32_t)(s * STAGE_BYTES);
        const uint64_t db = gmma_desc_sw128(st + (uint32_t)A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int m = 0; m < MT; ++m) {
            const uint64_t da = gmma_desc_sw128(st + (uint32_t)(m * A_TILE_BYTES) + g_off);
            // a 256-wide tile is issued as two 128-wide halves: the m64n256 fragment is the two m64n128 fragments side by side, and
            // one instruction with 128 live accumulators does not fit the register budget
            constexpr int NW = BN > 128 ? 128 : BN;
#pragma unroll
            for (int nb = 0; nb < BN / NW; ++nb) {
                float (&dh)[NW / 2] = *reinterpret_cast<float (*)[NW / 2]>(&d[m][nb * (NW / 2)]);
#pragma unroll
                for (int k = 0; k < BLOCK_K / 16; ++k)
                    wgmma_bf16<NW>(dh, da + (uint64_t)(k * 2), db + (uint64_t)(nb * NW * 8 + k * 2), (i > 0 || k > 0) ? 1u : 0u);
            }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
}
// registers -> the shared accumulator tile [MT * 128][BN], then one arrival per consumer warp on `bar`
template <int BN, int MT>
OA_DEVINL void wg_acc_publish(float* acc, const float (&d)[MT][BN / 2], uint64_t* bar) {
    const int g = threadIdx.x >> 7;
#pragma unroll
    for (int m = 0; m < MT; ++m) acc_store_frag<BN>(acc, m * BLOCK_M + g * 64, d[m]);
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}
constexpr int CONSUMER_WARPS = 8;

template <int BN>
struct GemmCfg {
    static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;              // 16 KB
    static constexpr int B_BYTES = BN * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int ACC_BYTES = BLOCK_M * BN * 4;
    // the fp32 accumulator tile shares the 227 KB with the ring; one CTA per SM at every width (288 threads x 168 registers)
    static constexpr int STAGES = BN >= 256 ? 2 : 4;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 1024 /*align*/ + 256 /*barriers*/;
    static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory budget of one CTA");
};

template <int BN, int EPI>
__global__ void OA_GEMM_REGS gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                      const __grid_constant__ CUtensorMap tmB,
                                                                      const GemmParams p) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* acc = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::ACC_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* acc_bar = empty_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    // Grouped rasterisation: CTAs walk bands of RASTER_GROUP_M row tiles, M fastest inside a band, so a band of A
    // (16 x 128 rows) stays L2-resident while each B tile is streamed from HBM once per band instead of once per row tile.
    int n_blk, m_blk;
    {
        const int n_tiles = (p.N + BN - 1) / BN, m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
        const int per_band = RASTER_GROUP_M * n_tiles;
        const int band = (int)blockIdx.x / per_band, within = (int)blockIdx.x - band * per_band;
        const int m0 = band * RASTER_GROUP_M;
        const int rows = (m_tiles - m0) < RASTER_GROUP_M ? (m_tiles - m0) : RASTER_GROUP_M;
        m_blk = m0 + within % rows; n_blk = within / rows;
    }
    const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;

    if (warp == PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_WARPS); }
        mbar_init(acc_bar, CONSUMER_WARPS);
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch();

    if (warp >= PRODUCER_WARP) {
        if (warp == PRODUCER_WARP && lane == 0) {
            // weights (B) are written by no kernel of the chain: fill the ring with them BEFORE waiting for the predecessor
            const int pre = num_kb < STAGES ? num_kb : STAGES;
            for (int kb = 0; kb < pre; ++kb) {
                mbar_expect_tx(&full_bar[kb], Cfg::STAGE_BYTES);
                tma_load_2d(smem + kb * Cfg::STAGE_BYTES + Cfg::A_BYTES, &tmB, &full_bar[kb], kb * BLOCK_K, n_blk * BN, kEvictFirst);
            }
            griddep_wait();
            for (int kb = 0; kb < pre; ++kb)
                tma_load_2d(smem + kb * Cfg::STAGE_BYTES, &tmA, &full_bar[kb], kb * BLOCK_K, m_blk * BLOCK_M, kEvictLast);
            int s = pre == STAGES ? 0 : pre; uint32_t ph = pre == STAGES ? 1 : 0;
            for (int kb = pre; kb < num_kb; ++kb) {
                mbar_wait(&empty_bar[s], ph ^ 1);
                uint8_t* a_dst = smem + s * Cfg::STAGE_BYTES;
                uint8_t* b_dst = a_dst + Cfg::A_BYTES;
                mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
                tma_load_2d(a_dst, &tmA, &full_bar[s], kb * BLOCK_K, m_blk * BLOCK_M, kEvictLast);
                tma_load_2d(b_dst, &tmB, &full_bar[s], kb * BLOCK_K, n_blk * BN, kEvictFirst);
                if (++s == STAGES) { s = 0; ph ^= 1; }
            }
        }
    } else if (warp < CONSUMER_WARPS) {
        float d[1][BN / 2] = {};
        int s = 0; uint32_t ph = 0;
        wg_mma_run<BN, 1, STAGES, Cfg::STAGE_BYTES, Cfg::A_BYTES, Cfg::A_BYTES>(d, smem, full_bar, s, ph, num_kb);
        wg_acc_publish<BN, 1>(acc, d, acc_bar);
        if (warp >= 4) return;
        // ---------------- epilogue: warpgroup 0, rows [32q, 32q + 32) with q = warp % 4 ----------------
        const int q = warp & 3;
        const int row = m_blk * BLOCK_M + q * 32 + lane;
        const bool row_ok = row < p.M;
        griddep_wait();                   // bias/residual reads and every store below come after the predecessor grid
        mbar_wait(acc_bar, 0);
        float best_v = -INFINITY; int best_i = 0x7fffffff;
        const uint32_t* mask_row = nullptr;
        if (EPI == EPI_LOGITS && row_ok && p.mask_slot) { const int ms = p.mask_slot[row]; if (ms >= 0) mask_row = p.mask_table + (size_t)ms * p.mask_words; }
#pragma unroll 1
        for (int c = 0; c < BN; c += 32) {
            uint32_t v[32];
            acc_ld32(acc, BN, q * 32 + lane, c, v);
            const int col0 = n_blk * BN + c;
            if (EPI == EPI_STORE) {
                if (row_ok) {
                    uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo;
                    const uint16_t* bias = reinterpret_cast<const uint16_t*>(p.bias);
#pragma unroll
                    for (int j = 0; j < 32; j += 8) {
                        if (col0 + j < p.N) {
                            float f[8];
#pragma unroll
                            for (int i = 0; i < 8; ++i) f[i] = __uint_as_float(v[j + i]);
                            if (bias) {
                                uint4 bb = *reinterpret_cast<const uint4*>(bias + col0 + j);
                                f[0] += bf16lo(bb.x); f[1] += bf16hi(bb.x); f[2] += bf16lo(bb.y); f[3] += bf16hi(bb.y);
                                f[4] += bf16lo(bb.z); f[5] += bf16hi(bb.z); f[6] += bf16lo(bb.w); f[7] += bf16hi(bb.w);
                            }
                            uint4 o;
                            o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]);
                            o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
                            *reinterpret_cast<uint4*>(orow + col0 + j) = o;
                        }
                    }
                }
            } else if (EPI == EPI_RESID) {
                if (row_ok) {
                    uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo;
                    const uint16_t* rrow = reinterpret_cast<const uint16_t*>(p.resid) + (size_t)row * p.ldr;
#pragma unroll
                    for (int j = 0; j < 32; j += 8) {
                        if (col0 + j < p.N) {
                            uint4 rr = *reinterpret_cast<const uint4*>(rrow + col0 + j);
                            uint4 o;
                            o.x = pack_bf16x2(__uint_as_float(v[j + 0]) + bf16lo(rr.x), __uint_as_float(v[j + 1]) + bf16hi(rr.x));
                            o.y = pack_bf16x2(__uint_as_float(v[j + 2]) + bf16lo(rr.y), __uint_as_float(v[j + 3]) + bf16hi(rr.y));
                            o.z = pack_bf16x2(__uint_as_float(v[j + 4]) + bf16lo(rr.z), __uint_as_float(v[j + 5]) + bf16hi(rr.z));
                            o.w = pack_bf16x2(__uint_as_float(v[j + 6]) + bf16lo(rr.w), __uint_as_float(v[j + 7]) + bf16hi(rr.w));
                            *reinterpret_cast<uint4*>(orow + col0 + j) = o;
                        }
                    }
                }
            } else if (EPI == EPI_SWIGLU) {
                // columns [c, c+16) = gate, [c+16, c+32) = up for output features (col0/2 .. col0/2+15)
                if (row_ok && col0 < p.N) {
                    uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo + (col0 >> 1);
                    float f[16];
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        float g = __uint_as_float(v[i]), u = __uint_as_float(v[16 + i]);
                        f[i] = __fdividef(g, 1.0f + __expf(-g)) * u;
                    }
                    uint4 o0, o1;
                    o0.x = pack_bf16x2(f[0], f[1]); o0.y = pack_bf16x2(f[2], f[3]); o0.z = pack_bf16x2(f[4], f[5]); o0.w = pack_bf16x2(f[6], f[7]);
                    o1.x = pack_bf16x2(f[8], f[9]); o1.y = pack_bf16x2(f[10], f[11]); o1.z = pack_bf16x2(f[12], f[13]); o1.w = pack_bf16x2(f[14], f[15]);
                    *reinterpret_cast<uint4*>(orow) = o0;
                    *reinterpret_cast<uint4*>(orow + 8) = o1;
                }
            } else {  // EPI_LOGITS
                if (row_ok) {
                    if (mask_row) {
                        // grammar-constrained row: only token ids allowed in this sequence's automaton state compete.  The 32 columns of
                        // this chunk are 32 consecutive global ids: at most two words of the bitset.
                        const uint32_t g0 = (uint32_t)(p.col_offset + col0);
                        const uint32_t w0 = (g0 >> 5) < (uint32_t)p.mask_words ? __ldg(mask_row + (g0 >> 5)) : 0u;
                        const uint32_t w1 = ((g0 & 31u) && (g0 >> 5) + 1 < (uint32_t)p.mask_words) ? __ldg(mask_row + (g0 >> 5) + 1) : 0u;
                        const uint32_t bits = (g0 & 31u) ? __funnelshift_r(w0, w1, g0 & 31u) : w0;
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            float f = __uint_as_float(v[j]);
                            if (((bits >> j) & 1u) && col0 + j < p.N && f > best_v) { best_v = f; best_i = col0 + j; }
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            float f = __uint_as_float(v[j]);
                            if (col0 + j < p.N && f > best_v) { best_v = f; best_i = col0 + j; }
                        }
                    }
                    if (p.logits) {
                        float* lrow = p.logits + (size_t)row * p.ldl;
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            if (col0 + j < p.N)
                                *reinterpret_cast<float4*>(lrow + col0 + j) =
                                    make_float4(__uint_as_float(v[j]), __uint_as_float(v[j + 1]), __uint_as_float(v[j + 2]), __uint_as_float(v[j + 3]));
                        }
                    }
                }
            }
        }
        if (EPI == EPI_LOGITS && row_ok) {
            const int n_tiles = (p.N + BN - 1) / BN;
            p.amax_val[(size_t)row * n_tiles + n_blk] = best_v;
            p.amax_idx[(size_t)row * n_tiles + n_blk] = best_i;
        }
    }
}

int gemm_n_tiles(int N, int block_n) { return (N + block_n - 1) / block_n; }

template <int BN, int EPI>
static cudaError_t launch_one(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, cudaStream_t stream) {
    using Cfg = GemmCfg<BN>;
    auto kern = gemm_wgmma_kernel<BN, EPI>;
    static bool attr_done[16] = {};
    { cudaError_t e = ensure_dynamic_smem(kern, Cfg::SMEM_BYTES, attr_done); if (e != cudaSuccess) return e; }
    dim3 grid(((p.N + BN - 1) / BN) * ((p.M + BLOCK_M - 1) / BLOCK_M), 1, 1);
    return launch_k(kern, grid, dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, *tmA, *tmB, p);
}

template <int BN>
static cudaError_t launch_bn(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, int epi, cudaStream_t s) {
    switch (epi) {
        case EPI_STORE: return launch_one<BN, EPI_STORE>(tmA, tmB, p, s);
        case EPI_RESID: return launch_one<BN, EPI_RESID>(tmA, tmB, p, s);
        case EPI_SWIGLU: return launch_one<BN, EPI_SWIGLU>(tmA, tmB, p, s);
        case EPI_LOGITS: return launch_one<BN, EPI_LOGITS>(tmA, tmB, p, s);
    }
    return cudaErrorInvalidValue;
}

static bool persistent_disabled();
static constexpr int PERSIST_BN = 128;      // 64 accumulator registers per consumer thread: no spills, and a 4-deep ring next to the 64 KB tile
static int sm_count_cached();
static long long persistent_min_tiles();
template <int EPI>
static cudaError_t launch_persistent(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, cudaStream_t stream);

cudaError_t launch_gemm(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, int epilogue, int block_n,
                        cudaStream_t stream) {
    if (p.M <= 0 || p.N <= 0 || p.K <= 0 || (p.N % 8) != 0 || (p.K % 8) != 0) return cudaErrorInvalidValue;
    if (epilogue == EPI_SWIGLU && (p.N % 32) != 0) return cudaErrorInvalidValue;
    // large-M (prefill) shapes with the persistent kernel's tile go to it (epilogue overlapped with the next tile); tmB's box is block_n rows
    if (block_n == PERSIST_BN && epilogue != EPI_LOGITS && !persistent_disabled() &&
        (long long)((p.N + PERSIST_BN - 1) / PERSIST_BN) * ((p.M + BLOCK_M - 1) / BLOCK_M) >= persistent_min_tiles()) {
        switch (epilogue) {
            case EPI_STORE: return launch_persistent<EPI_STORE>(tmA, tmB, p, stream);
            case EPI_RESID: return launch_persistent<EPI_RESID>(tmA, tmB, p, stream);
            case EPI_SWIGLU: return launch_persistent<EPI_SWIGLU>(tmA, tmB, p, stream);
        }
    }
    switch (block_n) {
        case 32: return launch_bn<32>(tmA, tmB, p, epilogue, stream);
        case 64: return launch_bn<64>(tmA, tmB, p, epilogue, stream);
        case 128: return launch_bn<128>(tmA, tmB, p, epilogue, stream);
        case 256: return launch_bn<256>(tmA, tmB, p, epilogue, stream);
    }
    return cudaErrorInvalidValue;
}

// =============================================================================================
// persistent tile GEMM (prefill, M > 128): one CTA per SM loops over 128 x 128 tiles in grouped raster order; warpgroup 1 runs the
// wgmma main loop of tile i+1 while warpgroup 0 stores tile i.
// =============================================================================================
struct PersistCfg {
    static constexpr int BN = PERSIST_BN;
    static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2, B_BYTES = BN * BLOCK_K * 2, STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = 4;
    static constexpr int ACC_BYTES = BLOCK_M * BN * 4;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 1024 + 256;
    static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory budget of one CTA");
};

OA_DEVINL void raster_tile(int idx, int m_tiles, int n_tiles, int& m_blk, int& n_blk) {
    const int per_band = RASTER_GROUP_M * n_tiles;
    const int band = idx / per_band, within = idx - band * per_band;
    const int m0 = band * RASTER_GROUP_M;
    const int rows = (m_tiles - m0) < RASTER_GROUP_M ? (m_tiles - m0) : RASTER_GROUP_M;
    m_blk = m0 + within % rows; n_blk = within / rows;
}

template <int EPI>
__global__ void OA_GEMM_REGS gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                            const __grid_constant__ CUtensorMap tmB,
                                                                            const GemmParams p) {
    using Cfg = PersistCfg;
    constexpr int BN = Cfg::BN, STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* acc = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::ACC_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* acc_full = empty_bar + STAGES;
    uint64_t* acc_empty = acc_full + 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tiles = (p.N + BN - 1) / BN, m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
    const int total_tiles = n_tiles * m_tiles;
    const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;

    if (warp == PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_WARPS); }
        mbar_init(acc_full, CONSUMER_WARPS); mbar_init(acc_empty, 4);
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch();

    if (warp >= PRODUCER_WARP) {
        if (warp == PRODUCER_WARP && lane == 0) {
            griddep_wait();
            int s = 0; uint32_t ph = 0;
            for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                int m_blk, n_blk; raster_tile(t, m_tiles, n_tiles, m_blk, n_blk);
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* a_dst = smem + s * Cfg::STAGE_BYTES;
                    mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
                    tma_load_2d(a_dst, &tmA, &full_bar[s], kb * BLOCK_K, m_blk * BLOCK_M, kEvictNormal);
                    tma_load_2d(a_dst + Cfg::A_BYTES, &tmB, &full_bar[s], kb * BLOCK_K, n_blk * BN, kEvictNormal);
                    if (++s == STAGES) { s = 0; ph ^= 1; }
                }
            }
        }
    } else if (warp < CONSUMER_WARPS) {
        int s = 0; uint32_t ph = 0, it = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++it) {
            float d[1][BN / 2] = {};
            wg_mma_run<BN, 1, STAGES, Cfg::STAGE_BYTES, Cfg::A_BYTES, Cfg::A_BYTES>(d, smem, full_bar, s, ph, num_kb);
            mbar_wait(acc_empty, (it & 1) ^ 1);      // the epilogue has drained the previous tile
            wg_acc_publish<BN, 1>(acc, d, acc_full);
            if (warp >= 4) continue;
            // ---------------- epilogue: warpgroup 0 ----------------
            const int q = warp & 3;
            griddep_wait();
            int m_blk, n_blk; raster_tile(t, m_tiles, n_tiles, m_blk, n_blk);
            mbar_wait(acc_full, it & 1);
            const int row_base = m_blk * BLOCK_M + q * 32;
#pragma unroll 1
            for (int cc = 0; cc < BN; cc += 32) {
                const int col0 = n_blk * BN + cc;
                if (EPI == EPI_SWIGLU) {
                    // chunk = 16 gate + 16 up columns -> 16 output features; lane = (row, 8-feature half)
                    const int h = lane & 1;
#pragma unroll
                    for (int i2 = 0; i2 < 2; ++i2) {
                        const int r = i2 * 16 + (lane >> 1), row = row_base + r;
                        const int ar = q * 32 + r, ac = cc + h * 8;
                        const float4 g0 = acc_ld4(acc, BN, ar, ac), g1 = acc_ld4(acc, BN, ar, ac + 4);
                        const float4 u0 = acc_ld4(acc, BN, ar, ac + 16), u1 = acc_ld4(acc, BN, ar, ac + 20);
                        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
                        const float uu[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
                        float f[8];
#pragma unroll
                        for (int k = 0; k < 8; ++k) f[k] = __fdividef(gg[k], 1.0f + __expf(-gg[k])) * uu[k];
                        if (row < p.M && col0 < p.N) {
                            uint4 o; o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]); o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
                            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo + (col0 >> 1) + h * 8) = o;
                        }
                    }
                } else {
                    // lane = (row, 8-column group): 8 rows x 64 B per store instruction
                    const int c8 = (lane & 3) * 8, col = col0 + c8;
#pragma unroll
                    for (int i4 = 0; i4 < 4; ++i4) {
                        const int r = i4 * 8 + (lane >> 2), row = row_base + r;
                        const float4 a0 = acc_ld4(acc, BN, q * 32 + r, cc + c8), a1 = acc_ld4(acc, BN, q * 32 + r, cc + c8 + 4);
                        float f[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                        if (row < p.M && col < p.N) {
                            if (EPI == EPI_STORE) {
                                if (p.bias) {
                                    const uint4 bb = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.bias) + col);
                                    f[0] += bf16lo(bb.x); f[1] += bf16hi(bb.x); f[2] += bf16lo(bb.y); f[3] += bf16hi(bb.y);
                                    f[4] += bf16lo(bb.z); f[5] += bf16hi(bb.z); f[6] += bf16lo(bb.w); f[7] += bf16hi(bb.w);
                                }
                            } else {
                                const uint4 rr = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.resid) + (size_t)row * p.ldr + col);
                                f[0] += bf16lo(rr.x); f[1] += bf16hi(rr.x); f[2] += bf16lo(rr.y); f[3] += bf16hi(rr.y);
                                f[4] += bf16lo(rr.z); f[5] += bf16hi(rr.z); f[6] += bf16lo(rr.w); f[7] += bf16hi(rr.w);
                            }
                            uint4 o; o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]); o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
                            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo + col) = o;
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(acc_empty);
        }
    }
}

static bool persistent_disabled() { static const bool off = [] { const char* e = std::getenv("OA_GEMM_PERSISTENT"); return e && e[0] == '0'; }(); return off; }
// tests lower the threshold (OA_GEMM_PERSISTENT_MIN_TILES=1) to drive tiny shapes through the persistent kernel
static long long persistent_min_tiles() { const char* e = std::getenv("OA_GEMM_PERSISTENT_MIN_TILES"); return e ? std::atoll(e) : 2LL * sm_count_cached(); }
static int sm_count_cached() {
    static int n = 0;
    if (n == 0) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
    return n;
}

template <int EPI>
static cudaError_t launch_persistent(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, cudaStream_t stream) {
    auto kern = gemm_persistent_kernel<EPI>;
    static bool attr_done[16] = {};
    { cudaError_t e = ensure_dynamic_smem(kern, PersistCfg::SMEM_BYTES, attr_done); if (e != cudaSuccess) return e; }
    const int tiles = ((p.N + PersistCfg::BN - 1) / PersistCfg::BN) * ((p.M + BLOCK_M - 1) / BLOCK_M);
    const int grid = tiles < sm_count_cached() ? tiles : sm_count_cached();
    return launch_k(kern, dim3(grid), dim3(GEMM_THREADS), PersistCfg::SMEM_BYTES, stream, *tmA, *tmB, p);
}

// =============================================================================================
// stream-K (decode, M <= 128): persistent CTAs, balanced weight streaming, fp32 partials
// =============================================================================================
template <int BN, int MT>     // MT = 128-row tiles of A per unit (1: M <= 128, 2: M <= 256)
struct SkCfg {
    static constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;
    static constexpr int A_BYTES = MT * A_TILE_BYTES;
    static constexpr int B_BYTES = BN * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int ACC_BYTES = MT * BLOCK_M * BN * 4;
    static constexpr int STAGES_FIT = (SMEM_LIMIT - ACC_BYTES - 1024 - 256) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_FIT < 6 ? STAGES_FIT : 6;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 1024 + 256;
    static_assert(STAGES >= 2 && SMEM_BYTES <= SMEM_LIMIT, "shared memory budget of one CTA");
};

// Epilogues finished INSIDE the stream-K GEMM by the CTA that holds a tile's first k-block (FUSE != 0): it adds the other CTAs' published
// pieces to its own accumulator in CTA order (the stand-alone consumers' order: bit-identical sums) and writes the final bf16 result.
//   FUSE 1  gate/up : act = silu(gate) * up
//   FUSE 2  o / down: x += acc            (residual stream, bf16, in place)
//   FUSE 3  qkv     : (+ bias) -> bf16 -> RoPE -> q_out / paged K rows; V rows copied
struct SkFuse {
    uint16_t* act; int F; unsigned int* tile_flags;
    uint16_t* x; int ldx; int N;        // FUSE 2 (N = logical output columns; also the bound of FUSE 3)
    SkRopeArgs rope;                    // FUSE 3
};

template <int BN, int MT, int FUSE = 0>
__global__ void OA_GEMM_REGS gemm_streamk_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                         const __grid_constant__ CUtensorMap tmB, const int M,
                                                                         const StreamK sk, const SkFuse fz) {
    using Cfg = SkCfg<BN, MT>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* acc_s = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);    // accumulator tile [MT * 128][BN]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::ACC_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* acc_full = empty_bar + STAGES;
    uint64_t* acc_empty = acc_full + 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long c = blockIdx.x, G = gridDim.x;
    const long long u0 = c * sk.total / G, u1 = (c + 1) * sk.total / G;

    if (warp == PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_WARPS); }
        mbar_init(acc_full, CONSUMER_WARPS); mbar_init(acc_empty, 4);
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch();

    if (warp >= PRODUCER_WARP) {
        if (warp == PRODUCER_WARP && lane == 0) {
            // weights first: they depend on no predecessor, so the HBM stream starts while the previous kernel drains
            const int pre = (u1 - u0) < STAGES ? (int)(u1 - u0) : STAGES;
            for (int i = 0; i < pre; ++i) {
                const long long u = u0 + i;
                const int tile = (int)(u / sk.kb), kblk = (int)(u - (long long)tile * sk.kb);
                mbar_expect_tx(&full_bar[i], Cfg::STAGE_BYTES);
                tma_load_2d(smem + i * Cfg::STAGE_BYTES + Cfg::A_BYTES, &tmB, &full_bar[i], kblk * BLOCK_K, tile * BN, kEvictFirst);
            }
            // ... and pull the next weight tiles into L2 while the (L2-bound) predecessor still runs and HBM is idle
            {
                const long long pf_end = (u0 + pre + sk.l2_prefetch_units) < u1 ? (u0 + pre + sk.l2_prefetch_units) : u1;
                for (long long u = u0 + pre; u < pf_end; ++u) {
                    const int tile = (int)(u / sk.kb), kblk = (int)(u - (long long)tile * sk.kb);
                    tma_prefetch_l2_2d(&tmB, kblk * BLOCK_K, tile * BN);
                }
            }
            griddep_wait();
            for (int i = 0; i < pre; ++i) {
                const long long u = u0 + i;
                const int tile = (int)(u / sk.kb), kblk = (int)(u - (long long)tile * sk.kb);
#pragma unroll
                for (int m = 0; m < MT; ++m)
                    tma_load_2d(smem + i * Cfg::STAGE_BYTES + m * Cfg::A_TILE_BYTES, &tmA, &full_bar[i], kblk * BLOCK_K, m * BLOCK_M, kEvictLast);
            }
            int s = pre == STAGES ? 0 : pre; uint32_t ph = pre == STAGES ? 1 : 0;
            for (long long u = u0 + pre; u < u1; ++u) {
                const int tile = (int)(u / sk.kb), kblk = (int)(u - (long long)tile * sk.kb);
                mbar_wait(&empty_bar[s], ph ^ 1);
                uint8_t* a_dst = smem + s * Cfg::STAGE_BYTES;
                mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
#pragma unroll
                for (int m = 0; m < MT; ++m)
                    tma_load_2d(a_dst + m * Cfg::A_TILE_BYTES, &tmA, &full_bar[s], kblk * BLOCK_K, m * BLOCK_M, kEvictLast);
                tma_load_2d(a_dst + Cfg::A_BYTES, &tmB, &full_bar[s], kblk * BLOCK_K, tile * BN, kEvictFirst);
                if (++s == STAGES) { s = 0; ph ^= 1; }
            }
        }
    } else if (warp < CONSUMER_WARPS) {
        int s = 0; uint32_t ph = 0, seg = 0;
        for (long long u = u0; u < u1; ++seg) {
            const int tile = (int)(u / sk.kb);
            const long long uend = min(u1, (long long)(tile + 1) * sk.kb);
            float d[MT][BN / 2] = {};
            wg_mma_run<BN, MT, STAGES, Cfg::STAGE_BYTES, Cfg::A_TILE_BYTES, Cfg::A_BYTES>(d, smem, full_bar, s, ph, (int)(uend - u));
            mbar_wait(acc_empty, (seg & 1) ^ 1);      // the epilogue has drained the previous segment
            wg_acc_publish<BN, MT>(acc_s, d, acc_full);
            if (warp >= 4) { u = uend; continue; }
            // ---------------- epilogue: warpgroup 0 ----------------
            const int q = warp & 3;
            griddep_wait();                   // the predecessor may still be reading the partial workspace
            mbar_wait(acc_full, seg & 1);
            if constexpr (FUSE == 2 || FUSE == 3) {
                // Same publish / finish protocol as the SwiGLU epilogue below (see there for why the finishing CTA never waits on a
                // waiting CTA); only what the finisher does with the summed 128 x 128 tile differs.
                uint32_t cf, cl;
                sk_tile_ctas(sk, (uint32_t)tile, cf, cl);
                const int c_first = (int)cf, c_last = (int)cl;
                const int row = q * 32 + lane;
                unsigned int* flag = fz.tile_flags + tile;
                if ((int)c == c_first) {
                    const int n_other = c_last - c_first;
                    if (n_other > 0) {
                        if (threadIdx.x == EPI_WARP0 * 32) { grid_counter_wait32(flag, (unsigned int)n_other); *flag = 0u; }
                        asm volatile("bar.sync 1, 128;" ::: "memory");
                    }
                    const float* other = sk.ws + (size_t)(c_first + 1 + tile) * (BLOCK_M * BN) + row;
                    const bool live = row < M;
                    // acc[0..32) = this row's sums of columns [mc, mc+32) of the tile: own accumulator, then the other pieces in CTA order
                    auto acc_chunk = [&](int mc, float (&acc)[32]) {
                        uint32_t v[32];
                        acc_ld32(acc_s, BN, row, mc, v);
#pragma unroll
                        for (int j = 0; j < 32; ++j) acc[j] = 0.f + __uint_as_float(v[j]);      // "0 +" as in sk_sum8
                        for (int o = 0; o < n_other; ++o) {
                            const float* pc = other + (size_t)o * (BLOCK_M * BN) + (size_t)mc * BLOCK_M;
                            float t[32];
#pragma unroll
                            for (int j = 0; j < 32; ++j) t[j] = live ? __ldcg(pc + (size_t)j * BLOCK_M) : 0.f;
#pragma unroll
                            for (int j = 0; j < 32; ++j) acc[j] += t[j];
                        }
                    };
                    if constexpr (FUSE == 2) {
#pragma unroll 1
                        for (int mc = 0; mc < BN; mc += 32) {
                            const int col0 = tile * BN + mc;
                            if (col0 >= fz.N) break;
                            float acc[32];
                            acc_chunk(mc, acc);
                            if (live) {
                                uint4* xr = reinterpret_cast<uint4*>(fz.x + (size_t)row * fz.ldx + col0);
#pragma unroll
                                for (int h = 0; h < 4; ++h) {
                                    const uint4 xo = __ldcg(xr + h);
                                    uint4 xn;
                                    xn.x = pack_bf16x2(bf16lo(xo.x) + acc[8 * h + 0], bf16hi(xo.x) + acc[8 * h + 1]); xn.y = pack_bf16x2(bf16lo(xo.y) + acc[8 * h + 2], bf16hi(xo.y) + acc[8 * h + 3]);
                                    xn.z = pack_bf16x2(bf16lo(xo.z) + acc[8 * h + 4], bf16hi(xo.z) + acc[8 * h + 5]); xn.w = pack_bf16x2(bf16lo(xo.w) + acc[8 * h + 6], bf16hi(xo.w) + acc[8 * h + 7]);
                                    xr[h] = xn;
                                }
                            }
                        }
                    } else {
                        const SkRopeArgs& a = fz.rope;
                        const int D = a.D, half = D >> 1;
                        int pos = 0, page = 0, off = 0;
                        if (live) { pos = a.positions[row]; const int slot = a.slots[row]; page = slot / a.page_size; off = slot - page * a.page_size; }
                        auto finish32 = [&](int col, float (&v)[32]) {          // + bias, round: the projection output is a bf16 tensor (sk_finish8_bf16)
                            if (a.bias) {
#pragma unroll
                                for (int h = 0; h < 4; ++h) {
                                    const uint4 bb = *reinterpret_cast<const uint4*>(a.bias + col + 8 * h);
                                    v[8 * h + 0] += bf16lo(bb.x); v[8 * h + 1] += bf16hi(bb.x); v[8 * h + 2] += bf16lo(bb.y); v[8 * h + 3] += bf16hi(bb.y);
                                    v[8 * h + 4] += bf16lo(bb.z); v[8 * h + 5] += bf16hi(bb.z); v[8 * h + 6] += bf16lo(bb.w); v[8 * h + 7] += bf16hi(bb.w);
                                }
                            }
#pragma unroll
                            for (int k = 0; k < 32; ++k) v[k] = bf16_bits_to_f32(f32_to_bf16_bits(v[k]));
                        };
                        auto store32 = [&](uint16_t* dst, const float (&v)[32]) {
#pragma unroll
                            for (int h = 0; h < 4; ++h) {
                                uint4 o;
                                o.x = pack_bf16x2(v[8 * h + 0], v[8 * h + 1]); o.y = pack_bf16x2(v[8 * h + 2], v[8 * h + 3]);
                                o.z = pack_bf16x2(v[8 * h + 4], v[8 * h + 5]); o.w = pack_bf16x2(v[8 * h + 6], v[8 * h + 7]);
                                reinterpret_cast<uint4*>(dst)[h] = o;
                            }
                        };
#pragma unroll 1
                        for (int mc = 0; mc < BN; mc += 32) {
                            const int col0 = tile * BN + mc;
                            if (col0 >= fz.N) break;
                            const int head = col0 / D, i0 = col0 - head * D;
                            if (head >= a.nh + a.nkv) {                    // V: straight copy into the V plane
                                float vv[32];
                                acc_chunk(mc, vv);
                                finish32(col0, vv);
                                if (live) store32(a.kv_base + (size_t)(a.v_plane_row0 + ((int64_t)page * a.nkv + (head - a.nh - a.nkv)) * a.page_size + off) * D + i0, vv);
                                continue;
                            }
                            if (i0 >= half) continue;                       // the high half is rotated together with its low partner
                            float av[32], bv[32];
                            acc_chunk(mc, av);
                            acc_chunk(mc + half, bv);                       // same tile: BN is a multiple of D
                            finish32(col0, av);
                            finish32(col0 + half, bv);
                            if (live) {
                                const float* cr = a.rope_cos + (size_t)pos * half + i0;
                                const float* sr = a.rope_sin + (size_t)pos * half + i0;
                                float ra[32], rb[32];
#pragma unroll
                                for (int h = 0; h < 8; ++h) {
                                    const float4 c4 = *reinterpret_cast<const float4*>(cr + 4 * h), s4 = *reinterpret_cast<const float4*>(sr + 4 * h);
                                    const float cv[4] = {c4.x, c4.y, c4.z, c4.w}, sv[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
                                    for (int k = 0; k < 4; ++k) {
                                        ra[4 * h + k] = av[4 * h + k] * cv[k] - bv[4 * h + k] * sv[k];
                                        rb[4 * h + k] = bv[4 * h + k] * cv[k] + av[4 * h + k] * sv[k];
                                    }
                                }
                                uint16_t* dst;
                                if (head < a.nh) dst = a.q_out + (size_t)row * a.nh * D + (size_t)head * D;
                                else dst = a.kv_base + (size_t)(a.k_plane_row0 + ((int64_t)page * a.nkv + (head - a.nh)) * a.page_size + off) * D;
                                store32(dst + i0, ra);
                                store32(dst + i0 + half, rb);
                            }
                        }
                    }
                } else {
                    float* dst = sk.ws + (size_t)(c + tile) * (BLOCK_M * BN) + row;
#pragma unroll 1
                    for (int mc = 0; mc < BN; mc += 32) {
                        uint32_t v[32];
                        acc_ld32(acc_s, BN, row, mc, v);
                        if (row < M) {
#pragma unroll
                            for (int j = 0; j < 32; ++j) dst[(size_t)(mc + j) * BLOCK_M] = __uint_as_float(v[j]);
                        }
                    }
                    __threadfence();
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    if (threadIdx.x == EPI_WARP0 * 32) atomicAdd(flag, 1u);
                }
            } else if constexpr (FUSE == 1) {
                // Pieces of this tile live in CTAs c_first..c_last (same arithmetic as sk_sum8).  The CTA holding the FIRST k-block
                // finishes the tile: it reaches this segment last (it is the tail of its unit range, while the other pieces are the
                // HEAD of their CTAs' ranges), adds the published pieces to its accumulator in CTA order — the stand-alone
                // consumer's order, so results are bit-identical — and writes silu(gate)*up.  Private piece layout: [col][row],
                // so that publisher stores and finisher loads are one full 128-byte line per warp instruction.
                uint32_t cf, cl;
                sk_tile_ctas(sk, (uint32_t)tile, cf, cl);
                const int c_first = (int)cf, c_last = (int)cl;
                const int row = q * 32 + lane;
                unsigned int* flag = fz.tile_flags + tile;
                if ((int)c == c_first) {
                    const int n_other = c_last - c_first;
                    if (n_other > 0) {
                        if (threadIdx.x == EPI_WARP0 * 32) { grid_counter_wait32(flag, (unsigned int)n_other); *flag = 0u; }
                        asm volatile("bar.sync 1, 128;" ::: "memory");
                    }
                    const float* other = sk.ws + (size_t)(c_first + 1 + tile) * (BLOCK_M * BN) + row;
                    uint16_t* act_row = fz.act + (size_t)row * fz.F;
                    const bool live = row < M;
                    float t[2][32];
                    auto load_piece = [&](float (&dst)[32], const float* base, int mc) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) dst[j] = live ? __ldcg(base + (size_t)(mc + j) * BLOCK_M) : 0.f;
                    };
                    if (n_other > 0) load_piece(t[0], other, 0);
#pragma unroll
                    for (int k4 = 0; k4 < BN / 32; ++k4) {
                        const int mc = k4 * 32;
                        if (n_other > 0 && k4 + 1 < BN / 32) load_piece(t[(k4 + 1) & 1], other, mc + 32);      // next chunk's piece is in flight during this chunk's math
                        uint32_t v[32];
                        acc_ld32(acc_s, BN, row, mc, v);
                        float acc[32];
#pragma unroll
                        for (int j = 0; j < 32; ++j) acc[j] = 0.f + __uint_as_float(v[j]);      // "0 +" as in sk_sum8
                        if (n_other > 0) {
#pragma unroll
                            for (int j = 0; j < 32; ++j) acc[j] += t[k4 & 1][j];
                        }
                        for (int o = 1; o < n_other; ++o) {                                      // tiles cut into more than two pieces (small shapes)
                            float x[32];
                            load_piece(x, other + (size_t)o * (BLOCK_M * BN), mc);
#pragma unroll
                            for (int j = 0; j < 32; ++j) acc[j] += x[j];
                        }
                        const int f0 = (tile * BN + mc) >> 1;          // 32 physical columns = 16 gate + 16 up -> 16 outputs
                        if (live && f0 < fz.F) {
                            float f[16];
#pragma unroll
                            for (int k = 0; k < 16; ++k) f[k] = __fdividef(acc[k], 1.0f + __expf(-acc[k])) * acc[16 + k];
                            uint4 o0, o1;
                            o0.x = pack_bf16x2(f[0], f[1]); o0.y = pack_bf16x2(f[2], f[3]); o0.z = pack_bf16x2(f[4], f[5]); o0.w = pack_bf16x2(f[6], f[7]);
                            o1.x = pack_bf16x2(f[8], f[9]); o1.y = pack_bf16x2(f[10], f[11]); o1.z = pack_bf16x2(f[12], f[13]); o1.w = pack_bf16x2(f[14], f[15]);
                            *reinterpret_cast<uint4*>(act_row + f0) = o0;
                            *reinterpret_cast<uint4*>(act_row + f0 + 8) = o1;
                        }
                    }
                } else {
                    float* dst = sk.ws + (size_t)(c + tile) * (BLOCK_M * BN) + row;
#pragma unroll 1
                    for (int mc = 0; mc < BN; mc += 32) {
                        uint32_t v[32];
                        acc_ld32(acc_s, BN, row, mc, v);
                        if (row < M) {
#pragma unroll
                            for (int j = 0; j < 32; ++j) dst[(size_t)(mc + j) * BLOCK_M] = __uint_as_float(v[j]);
                        }
                    }
                    __threadfence();
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    if (threadIdx.x == EPI_WARP0 * 32) atomicAdd(flag, 1u);
                }
            } else {
            // read the shared accumulator tile row-wise so that every global store instruction writes four full 128-byte lines
            // (8 lanes per row)
            const int r_sub = lane >> 3, c4 = (lane & 7) * 4;
#pragma unroll 1
            for (int mc = 0; mc < MT * BN; mc += 32) {
                const int m = mc / BN, cc = mc - m * BN;
                float* dst = sk.ws + ((size_t)(c + tile) * (MT * BLOCK_M) + m * BLOCK_M + q * 32) * BN;
#pragma unroll
                for (int it = 0; it < 8; ++it) {
                    const int r = it * 4 + r_sub;
                    const float4 val = acc_ld4(acc_s, BN, m * BLOCK_M + q * 32 + r, cc + c4);
                    if (m * BLOCK_M + q * 32 + r < M) *reinterpret_cast<float4*>(dst + (size_t)r * BN + cc + c4) = val;
                }
            }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(acc_empty);
            u = uend;
        }
    }
}

StreamK make_streamk(float* ws, int N, int K, int bn, int G, int rows) {
    StreamK sk{}; sk.ws = ws; sk.bn = bn; sk.rows = rows > 128 ? 256 : 128; sk.kb = (K + BLOCK_K - 1) / BLOCK_K; sk.n_tiles = (N + bn - 1) / bn;
    sk.total = (long long)sk.n_tiles * sk.kb; sk.G = (int)std::min<long long>(G, sk.total);
    sk.l2_prefetch_units = 0;
    return sk;
}
size_t streamk_ws_bytes(int N, int bn, int G, int rows) { return (size_t)(G + (N + bn - 1) / bn) * (rows > 128 ? 256 : 128) * bn * sizeof(float); }

template <int BN, int MT, int FUSE = 0>
static cudaError_t launch_sk(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, const StreamK& sk, cudaStream_t stream, SkFuse fz = SkFuse{}) {
    auto kern = gemm_streamk_kernel<BN, MT, FUSE>;
    static bool attr_done[16] = {};
    { cudaError_t e = ensure_dynamic_smem(kern, SkCfg<BN, MT>::SMEM_BYTES, attr_done); if (e != cudaSuccess) return e; }
    return launch_k(kern, dim3(sk.G), dim3(GEMM_THREADS), SkCfg<BN, MT>::SMEM_BYTES, stream, *tmA, *tmB, M, sk, fz);
}
cudaError_t launch_gemm_streamk_swiglu(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int F, int K, const StreamK& sk, void* act,
                                       unsigned int* tile_flags, cudaStream_t stream) {
    if (M <= 0 || M > BLOCK_M || sk.rows != 128 || sk.bn != 128 || (F % 16) != 0 || (K % 8) != 0 || !act || !tile_flags) return cudaErrorInvalidValue;
    if (sk.G > sm_count_cached()) return cudaErrorInvalidValue;      // finishing CTAs wait for publishing CTAs: all must be resident
    SkFuse fz{}; fz.act = reinterpret_cast<uint16_t*>(act); fz.F = F; fz.tile_flags = tile_flags;
    return launch_sk<128, 1, 1>(tmA, tmB, M, sk, stream, fz);
}
cudaError_t launch_gemm_streamk_resid(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, void* x, int ldx,
                                      unsigned int* tile_flags, cudaStream_t stream) {
    if (M <= 0 || M > BLOCK_M || sk.rows != 128 || sk.bn != 128 || (N % 32) != 0 || (K % 8) != 0 || !x || !tile_flags || (ldx % 8) != 0) return cudaErrorInvalidValue;
    if (sk.G > sm_count_cached()) return cudaErrorInvalidValue;      // finishing CTAs wait for publishing CTAs: all must be resident
    SkFuse fz{}; fz.tile_flags = tile_flags; fz.x = reinterpret_cast<uint16_t*>(x); fz.ldx = ldx; fz.N = N;
    return launch_sk<128, 1, 2>(tmA, tmB, M, sk, stream, fz);
}
cudaError_t launch_gemm_streamk_rope(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, const SkRopeArgs& rope,
                                     unsigned int* tile_flags, cudaStream_t stream) {
    if (M <= 0 || M > BLOCK_M || sk.rows != 128 || sk.bn != 128 || (K % 8) != 0 || !tile_flags) return cudaErrorInvalidValue;
    if ((rope.D != 64 && rope.D != 128) || N != (rope.nh + 2 * rope.nkv) * rope.D) return cudaErrorInvalidValue;      // BN must be a multiple of D; chunks of 32 never straddle a head
    if (sk.G > sm_count_cached()) return cudaErrorInvalidValue;
    SkFuse fz{}; fz.tile_flags = tile_flags; fz.N = N; fz.rope = rope;
    return launch_sk<128, 1, 3>(tmA, tmB, M, sk, stream, fz);
}
cudaError_t launch_gemm_streamk(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, cudaStream_t stream) {
    if (M <= 0 || M > sk.rows || (N % 8) != 0 || (K % 8) != 0) return cudaErrorInvalidValue;
    if (sk.rows == 256) return sk.bn == 128 ? launch_sk<128, 2>(tmA, tmB, M, sk, stream) : cudaErrorInvalidValue;
    if (sk.bn == 256) return launch_sk<256, 1>(tmA, tmB, M, sk, stream);
    if (sk.bn == 128) return launch_sk<128, 1>(tmA, tmB, M, sk, stream);      // more CTAs than SMs run in waves: the plain kernel never waits on another CTA
    if (sk.bn == 64) return launch_sk<64, 1>(tmA, tmB, M, sk, stream);       // half the partial bytes again; per-projection opt-in (sk_bn_o / sk_bn_down / sk_bn_qkv)
    return cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------
__global__ void argmax_reduce_kernel(const float* __restrict__ val, const int* __restrict__ idx, int M, int n_tiles,
                                     int32_t* __restrict__ out_ids, float* __restrict__ out_val) {
    const int row = blockIdx.x;
    griddep_launch(); griddep_wait();
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int t = threadIdx.x; t < n_tiles; t += blockDim.x) {
        float v = val[(size_t)row * n_tiles + t]; int i = idx[(size_t)row * n_tiles + t];
        if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, bv, o); int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    __shared__ float sv[8]; __shared__ int si[8];
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
            if (sv[w] > bv || (sv[w] == bv && si[w] < bi)) { bv = sv[w]; bi = si[w]; }
        out_ids[row] = bi == 0x7fffffff ? 0 : bi;
        if (out_val) out_val[row] = bv;
    }
}

cudaError_t launch_argmax_reduce(const float* amax_val, const int* amax_idx, int M, int n_tiles, int32_t* out_ids,
                                 float* out_val, cudaStream_t stream) {
    return launch_k(argmax_reduce_kernel, dim3(M), dim3(256), 0, stream, amax_val, amax_idx, M, n_tiles, out_ids, out_val);
}

}  // namespace oa
