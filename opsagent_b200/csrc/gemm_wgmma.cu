// gemm_wgmma.cu — C[M,N] = A[M,K] · B[N,K]^T for the QKV / O / gate-up / down / LM-head projections, on the pipeline of
// gemm_pipe.cuh (TMA producer warp, two wgmma consumer warpgroups).
//
// Tile kernel (one CTA = one 128 x BLOCK_N output tile): at the end of the tile the consumers write the accumulator into a swizzled fp32
// tile in shared memory (`acc_full`), from which warpgroup 0 runs the epilogue, one output row per thread (bias | residual add | SwiGLU |
// fp32 logits + row arg-max).  Decode (M <= 128) is weight-streaming and HBM-bound: B tiles are fetched with an evict-first L2 policy,
// the small A operand with evict-last.  K tails and M/N tails rely on TMA zero fill + predicated stores.
// FP8 instantiations (weight_dtype fp8_e4m3): e4m3 A and B with per-row fp32 scales, applied as a fragment enters the shared fp32 tile.
//
// The role of this file in the reference's terms: it is the arithmetic that sits behind
// llms.OpenAIClient.Chat (reference pkg/llms/openai.go:69-104) once the `local-cuda` provider replaces the
// remote HTTP server — see DESIGN.md §Kernels.
#include <algorithm>
#include <cstdlib>

#include "gemm_pipe.cuh"
#include "sk_consumers.cuh"

namespace oa {

// the fp32 tile shares the 227 KB with the ring; one CTA per SM at every width.  FP8: e4m3 operands (same bytes per unit, twice the K)
template <int BN, bool FP8 = false>
using GemmCfg = RingCfg<BN, 1, BN >= 256 ? 2 : 4, BLOCK_M * BN * 4, FP8>;

template <int BN, int EPI, bool FP8 = false>
__global__ void OA_GEMM_REGS gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                      const __grid_constant__ CUtensorMap tmB,
                                                                      const GemmParams p) {
    using Cfg = GemmCfg<BN, FP8>;
    extern __shared__ uint8_t smem_raw[];
    const Ring ring = ring_setup<Cfg>(smem_raw, &tmA, &tmB);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    int n_blk, m_blk;
    raster_tile((int)blockIdx.x, (p.M + BLOCK_M - 1) / BLOCK_M, (p.N + BN - 1) / BN, m_blk, n_blk);
    const int num_kb = (p.K + Cfg::KE - 1) / Cfg::KE;

    if (warp >= PRODUCER_WARP) {
        if (warp == PRODUCER_WARP && lane == 0) {
            auto unit = [&](int kb, int& kx, int& a_row, int& b_row) { kx = kb * Cfg::KE; a_row = m_blk * BLOCK_M; b_row = n_blk * BN; };
            ring_produce<Cfg, true>(ring, &tmA, &tmB, num_kb, unit, kEvictLast, kEvictFirst);
        }
    } else if (warp < CONSUMER_WARPS) {
        float d[1][BN / 2] = {};
        int s = 0; uint32_t ph = 0;
        wg_mma_run<Cfg>(d, ring, s, ph, num_kb);
        if constexpr (FP8) wg_scale_frag<BN, 1>(d, p.w8, m_blk * BLOCK_M, n_blk * BN, p.M, p.N);
        float* acc = ring.acc;
        wg_acc_publish<BN, 1>(acc, d, ring.acc_full);
        if (warp >= 4) return;
        // ---------------- epilogue: warpgroup 0, rows [32q, 32q + 32) with q = warp % 4 ----------------
        const int q = warp & 3;
        const int row = m_blk * BLOCK_M + q * 32 + lane;
        const bool row_ok = row < p.M;
        griddep_wait();                   // bias/residual reads and every store below come after the predecessor grid
        mbar_wait(ring.acc_full, 0);
        float best_v = -INFINITY; int best_i = 0x7fffffff;
        const uint32_t* mask_row = nullptr;
        if (EPI == EPI_LOGITS && row_ok && p.mask_slot) { const int ms = p.mask_slot[row]; if (ms >= 0) mask_row = p.mask_table + (size_t)ms * p.mask_words; }
#pragma unroll 1
        for (int c = 0; c < BN; c += 32) {
            uint32_t v[32];
            acc_ld32(acc, BN, q * 32 + lane, c, v);
            const int col0 = n_blk * BN + c;
            if (EPI == EPI_STORE || EPI == EPI_RESID) {
                if (row_ok) {
                    uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo;
#pragma unroll
                    for (int j = 0; j < 32; j += 8) {
                        if (col0 + j < p.N) {
                            float f[8];
#pragma unroll
                            for (int i = 0; i < 8; ++i) f[i] = __uint_as_float(v[j + i]);
                            if (EPI == EPI_STORE) {
                                if (p.bias) add_bf16x8(f, *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.bias) + col0 + j));
                            } else {
                                add_bf16x8(f, *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.resid) + (size_t)row * p.ldr + col0 + j));
                            }
                            *reinterpret_cast<uint4*>(orow + col0 + j) = pack_bf16x8(f);
                        }
                    }
                }
            } else if (EPI == EPI_SWIGLU) {
                // columns [c, c+16) = gate, [c+16, c+32) = up for output features (col0/2 .. col0/2+15)
                if (row_ok && col0 < p.N) {
                    uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo + (col0 >> 1);
                    float g[16], u[16];
#pragma unroll
                    for (int i = 0; i < 16; ++i) { g[i] = __uint_as_float(v[i]); u[i] = __uint_as_float(v[16 + i]); }
                    *reinterpret_cast<uint4*>(orow) = swiglu_bf16x8(g, u);
                    *reinterpret_cast<uint4*>(orow + 8) = swiglu_bf16x8(g + 8, u + 8);
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

template <int BN, int EPI, bool FP8 = false>
static cudaError_t launch_one(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, cudaStream_t stream) {
    const dim3 grid(((p.N + BN - 1) / BN) * ((p.M + BLOCK_M - 1) / BLOCK_M));
    return launch_gemm_kernel<gemm_wgmma_kernel<BN, EPI, FP8>>(grid, GemmCfg<BN, FP8>::SMEM_BYTES, stream, *tmA, *tmB, p);
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
// fp8 operands: the projections' epilogues only (the LM head stays bf16), N tiles up to 128 (the promoted fragment's registers)
template <int BN>
static cudaError_t launch_bn_fp8(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, int epi, cudaStream_t s) {
    switch (epi) {
        case EPI_STORE: return launch_one<BN, EPI_STORE, true>(tmA, tmB, p, s);
        case EPI_RESID: return launch_one<BN, EPI_RESID, true>(tmA, tmB, p, s);
        case EPI_SWIGLU: return launch_one<BN, EPI_SWIGLU, true>(tmA, tmB, p, s);
    }
    return cudaErrorInvalidValue;
}

static bool persistent_disabled();
static constexpr int PERSIST_BN = 128;      // 64 accumulator registers per consumer thread: no spills, and a 4-deep ring next to the 64 KB tile
static int sm_count_cached();
static long long persistent_min_tiles();
template <int EPI, bool FP8 = false>
static cudaError_t launch_persistent(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, cudaStream_t stream);

cudaError_t launch_gemm(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, int epilogue, int block_n,
                        cudaStream_t stream) {
    if (p.M <= 0 || p.N <= 0 || p.K <= 0 || (p.N % 8) != 0 || (p.K % 8) != 0) return cudaErrorInvalidValue;
    if (epilogue == EPI_SWIGLU && (p.N % 32) != 0) return cudaErrorInvalidValue;
    if (p.w8.a || p.w8.b) {
        if (!p.w8.a || !p.w8.b || (p.K % 16) != 0 || epilogue == EPI_LOGITS) return cudaErrorInvalidValue;
        if (block_n == PERSIST_BN && !persistent_disabled() &&
            (long long)((p.N + PERSIST_BN - 1) / PERSIST_BN) * ((p.M + BLOCK_M - 1) / BLOCK_M) >= persistent_min_tiles()) {
            switch (epilogue) {
                case EPI_STORE: return launch_persistent<EPI_STORE, true>(tmA, tmB, p, stream);
                case EPI_RESID: return launch_persistent<EPI_RESID, true>(tmA, tmB, p, stream);
                case EPI_SWIGLU: return launch_persistent<EPI_SWIGLU, true>(tmA, tmB, p, stream);
            }
        }
        switch (block_n) {
            case 32: return launch_bn_fp8<32>(tmA, tmB, p, epilogue, stream);
            case 64: return launch_bn_fp8<64>(tmA, tmB, p, epilogue, stream);
            case 128: return launch_bn_fp8<128>(tmA, tmB, p, epilogue, stream);
        }
        return cudaErrorInvalidValue;
    }
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
using PersistCfg = GemmCfg<PERSIST_BN>;      // (the fp8 ring has the same bytes)

template <int EPI, bool FP8 = false>
__global__ void OA_GEMM_REGS gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                            const __grid_constant__ CUtensorMap tmB,
                                                                            const GemmParams p) {
    using Cfg = GemmCfg<PERSIST_BN, FP8>;
    constexpr int BN = Cfg::BN;
    extern __shared__ uint8_t smem_raw[];
    const Ring ring = ring_setup<Cfg>(smem_raw, &tmA, &tmB);
    float* acc = ring.acc;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tiles = (p.N + BN - 1) / BN, m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
    const int total_tiles = n_tiles * m_tiles;
    const int num_kb = (p.K + Cfg::KE - 1) / Cfg::KE;

    if (warp >= PRODUCER_WARP) {
        if (warp == PRODUCER_WARP && lane == 0) {
            // this CTA's tiles blockIdx.x, blockIdx.x + gridDim.x, ... in turn, all k-blocks of each.  Units are visited once each, in
            // order, so the walk advances incrementally: the producer thread stays off the critical path of the compute-bound main loop.
            int t = blockIdx.x, kb = 0, m_blk = 0, n_blk = 0;
            if (t < total_tiles) raster_tile(t, m_tiles, n_tiles, m_blk, n_blk);
            auto unit = [&](int, int& kx, int& a_row, int& b_row) {
                kx = kb * Cfg::KE; a_row = m_blk * BLOCK_M; b_row = n_blk * BN;
                if (++kb == num_kb) { kb = 0; t += gridDim.x; if (t < total_tiles) raster_tile(t, m_tiles, n_tiles, m_blk, n_blk); }
            };
            const int my_tiles = ((int)blockIdx.x < total_tiles) ? (total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
            ring_produce<Cfg, false>(ring, &tmA, &tmB, my_tiles * num_kb, unit, kEvictNormal, kEvictNormal);
        }
    } else if (warp < CONSUMER_WARPS) {
        int s = 0; uint32_t ph = 0, it = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++it) {
            float d[1][BN / 2] = {};
            wg_mma_run<Cfg>(d, ring, s, ph, num_kb);
            int m_blk, n_blk; raster_tile(t, m_tiles, n_tiles, m_blk, n_blk);
            if constexpr (FP8) wg_scale_frag<BN, 1>(d, p.w8, m_blk * BLOCK_M, n_blk * BN, p.M, p.N);
            mbar_wait(ring.acc_empty, (it & 1) ^ 1);      // the epilogue has drained the previous tile
            wg_acc_publish<BN, 1>(acc, d, ring.acc_full);
            if (warp >= 4) continue;
            // ---------------- epilogue: warpgroup 0 ----------------
            const int q = warp & 3;
            griddep_wait();
            mbar_wait(ring.acc_full, it & 1);
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
                        if (row < p.M && col0 < p.N)
                            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo + (col0 >> 1) + h * 8) = swiglu_bf16x8(gg, uu);
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
                                if (p.bias) add_bf16x8(f, *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.bias) + col));
                            } else {
                                add_bf16x8(f, *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.resid) + (size_t)row * p.ldr + col));
                            }
                            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out) + (size_t)row * p.ldo + col) = pack_bf16x8(f);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(ring.acc_empty);
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

template <int EPI, bool FP8>
static cudaError_t launch_persistent(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p, cudaStream_t stream) {
    const int tiles = ((p.N + PersistCfg::BN - 1) / PersistCfg::BN) * ((p.M + BLOCK_M - 1) / BLOCK_M);
    const int grid = tiles < sm_count_cached() ? tiles : sm_count_cached();
    return launch_gemm_kernel<gemm_persistent_kernel<EPI, FP8>>(dim3(grid), PersistCfg::SMEM_BYTES, stream, *tmA, *tmB, p);
}

// =============================================================================================
// stream-K (decode, M <= 128): persistent CTAs, balanced weight streaming, fp32 partials
// =============================================================================================
template <int BN, int MT, bool FP8 = false>     // MT = 128-row tiles of A per unit (1: M <= 128, 2: M <= 256)
using SkCfg = RingCfg<BN, MT, ring_stages_fit(BN, MT, 6), MT * BLOCK_M * BN * 4, FP8>;

// Epilogues finished INSIDE the stream-K GEMM by the CTA that holds a tile's first k-block (FUSE != 0): it adds the other CTAs' published
// pieces to its own accumulator in CTA order (the stand-alone consumers' order: bit-identical sums) and writes the final bf16 result.
//   FUSE 1  gate/up : act = silu(gate) * up
//   FUSE 2  o / down: x += acc            (residual stream, bf16, in place)
//   FUSE 3  qkv     : (+ bias) -> bf16 -> RoPE -> q_out / paged K rows; V rows copied
struct SkFuse {
    uint16_t* act; int F; unsigned int* tile_flags;
    uint16_t* x; int ldx; int N;        // FUSE 2 (N = logical output columns; also the bound of FUSE 3 and of the fp8 column scales)
    SkRopeArgs rope;                    // FUSE 3
    W8Scales w8;                        // fp8 operands
};

// The fused finisher protocol.  Pieces of a tile live in CTAs c_first..c_last (sk_tile_ctas).  The CTA holding the FIRST k-block finishes
// the tile: it reaches this segment last (it is the tail of its unit range, while the other pieces are the HEAD of their CTAs' ranges), so
// it never waits on a CTA that is itself waiting.  Private piece layout: [col][row], so that publisher stores and finisher loads are one
// full 128-byte line per warp instruction.
// Finisher: wait until the n_other other CTAs of the tile have published their pieces, then re-arm the tile's counter.
OA_DEVINL void sk_wait_pieces(unsigned int* flag, int n_other) {
    if (n_other > 0) {
        if (threadIdx.x == EPI_WARP0 * 32) { grid_counter_wait32(flag, (unsigned int)n_other); *flag = 0u; }
        asm volatile("bar.sync 1, 128;" ::: "memory");
    }
}
// Publisher: this CTA's piece of `tile` (rows < M of the shared accumulator tile) -> its workspace slot, then count it on the tile's flag.
template <int BN>
OA_DEVINL void sk_publish_piece(const StreamK& sk, const float* acc_s, long long c, int tile, int row, int M, unsigned int* flag) {
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

template <int BN, int MT, int FUSE = 0, bool FP8 = false>
__global__ void OA_GEMM_REGS gemm_streamk_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                         const __grid_constant__ CUtensorMap tmB, const int M,
                                                                         const StreamK sk, const SkFuse fz) {
    using Cfg = SkCfg<BN, MT, FP8>;
    extern __shared__ uint8_t smem_raw[];
    const Ring ring = ring_setup<Cfg>(smem_raw, &tmA, &tmB);
    float* acc_s = ring.acc;                          // accumulator tile [MT * 128][BN]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long c = blockIdx.x, G = gridDim.x;
    const long long u0 = c * sk.total / G, u1 = (c + 1) * sk.total / G;

    if (warp >= PRODUCER_WARP) {
        if (warp == PRODUCER_WARP && lane == 0) {
            // weights first: the HBM stream starts, and the next weight tiles are pulled into L2, while the (L2-bound) predecessor drains
            auto unit = [&](int i, int& kx, int& a_row, int& b_row) {
                const long long u = u0 + i;
                const int tile = (int)(u / sk.kb), kblk = (int)(u - (long long)tile * sk.kb);
                kx = kblk * Cfg::KE; a_row = 0; b_row = tile * BN;
            };
            ring_produce<Cfg, true>(ring, &tmA, &tmB, (int)(u1 - u0), unit, kEvictLast, kEvictFirst, sk.l2_prefetch_units);
        }
    } else if (warp < CONSUMER_WARPS) {
        int s = 0; uint32_t ph = 0, seg = 0;
        for (long long u = u0; u < u1; ++seg) {
            const int tile = (int)(u / sk.kb);
            const long long uend = min(u1, (long long)(tile + 1) * sk.kb);
            float d[MT][BN / 2] = {};
            wg_mma_run<Cfg>(d, ring, s, ph, (int)(uend - u));
            if constexpr (FP8) wg_scale_frag<BN, MT>(d, fz.w8, 0, tile * BN, M, fz.N);
            mbar_wait(ring.acc_empty, (seg & 1) ^ 1);      // the epilogue has drained the previous segment
            wg_acc_publish<BN, MT>(acc_s, d, ring.acc_full);
            if (warp >= 4) { u = uend; continue; }
            // ---------------- epilogue: warpgroup 0 ----------------
            const int q = warp & 3;
            griddep_wait();                   // the predecessor may still be reading the partial workspace
            mbar_wait(ring.acc_full, seg & 1);
            if constexpr (FUSE != 0) {
                uint32_t cf, cl;
                sk_tile_ctas(sk, (uint32_t)tile, cf, cl);
                const int c_first = (int)cf, c_last = (int)cl;
                const int row = q * 32 + lane;
                unsigned int* flag = fz.tile_flags + tile;
                if ((int)c != c_first) {
                    sk_publish_piece<BN>(sk, acc_s, c, tile, row, M, flag);
                } else {
                    const int n_other = c_last - c_first;
                    sk_wait_pieces(flag, n_other);
                    const float* other = sk.ws + (size_t)(c_first + 1 + tile) * (BLOCK_M * BN) + row;
                    const bool live = row < M;
                    auto load_piece = [&](float (&dst)[32], const float* base, int mc) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) dst[j] = live ? __ldcg(base + (size_t)(mc + j) * BLOCK_M) : 0.f;
                    };
                    if constexpr (FUSE == 1) {
                        // gate/up: act = silu(gate) * up.  The first other piece of the next chunk is loaded during this chunk's math.
                        uint16_t* act_row = fz.act + (size_t)row * fz.F;
                        float t[2][32];
                        if (n_other > 0) load_piece(t[0], other, 0);
#pragma unroll
                        for (int k4 = 0; k4 < BN / 32; ++k4) {
                            const int mc = k4 * 32;
                            if (n_other > 0 && k4 + 1 < BN / 32) load_piece(t[(k4 + 1) & 1], other, mc + 32);
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
                                *reinterpret_cast<uint4*>(act_row + f0) = swiglu_bf16x8(acc, acc + 16);
                                *reinterpret_cast<uint4*>(act_row + f0 + 8) = swiglu_bf16x8(acc + 8, acc + 24);
                            }
                        }
                    } else {
                        // acc[0..32) = this row's sums of columns [mc, mc+32) of the tile: own accumulator, then the other pieces in CTA order
                        auto acc_chunk = [&](int mc, float (&acc)[32]) {
                            uint32_t v[32];
                            acc_ld32(acc_s, BN, row, mc, v);
#pragma unroll
                            for (int j = 0; j < 32; ++j) acc[j] = 0.f + __uint_as_float(v[j]);      // "0 +" as in sk_sum8
                            for (int o = 0; o < n_other; ++o) {
                                float t[32];
                                load_piece(t, other + (size_t)o * (BLOCK_M * BN), mc);
#pragma unroll
                                for (int j = 0; j < 32; ++j) acc[j] += t[j];
                            }
                        };
                        if constexpr (FUSE == 2) {
                            // o / down: x += acc (residual stream, bf16, in place)
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
                                        add_bf16x8(acc + 8 * h, __ldcg(xr + h));
                                        xr[h] = pack_bf16x8(acc + 8 * h);
                                    }
                                }
                            }
                        } else {
                            // qkv: (+ bias) -> bf16 -> RoPE -> q_out / paged K rows; V rows copied (sk_rope_item's arithmetic)
                            const SkRopeArgs& a = fz.rope;
                            const int D = a.D, half = D >> 1;
                            int pos = 0, page = 0, off = 0;
                            if (live) { pos = a.positions[row]; const int slot = a.slots[row]; page = slot / a.page_size; off = slot - page * a.page_size; }
#pragma unroll 1
                            for (int mc = 0; mc < BN; mc += 32) {
                                const int col0 = tile * BN + mc;
                                if (col0 >= fz.N) break;
                                const int head = col0 / D, i0 = col0 - head * D;
                                if (head >= a.nh + a.nkv) {                    // V: straight copy into the V plane
                                    float vv[32];
                                    acc_chunk(mc, vv);
#pragma unroll
                                    for (int h = 0; h < 4; ++h) qkv_finish8(a.bias, col0 + 8 * h, vv + 8 * h);
                                    if (live) {
#pragma unroll
                                        for (int h = 0; h < 4; ++h) kv_store8(a, row, head, page, off, i0 + 8 * h, pack_bf16x8(vv + 8 * h));
                                    }
                                    continue;
                                }
                                if (i0 >= half) continue;                       // the high half is rotated together with its low partner
                                float av[32], bv[32];
                                acc_chunk(mc, av);
                                acc_chunk(mc + half, bv);                       // same tile: BN is a multiple of D
#pragma unroll
                                for (int h = 0; h < 4; ++h) {
                                    qkv_finish8(a.bias, col0 + 8 * h, av + 8 * h);
                                    qkv_finish8(a.bias, col0 + half + 8 * h, bv + 8 * h);
                                }
                                if (live) {
                                    const float* cr = a.rope_cos + (size_t)pos * half + i0;
                                    const float* sr = a.rope_sin + (size_t)pos * half + i0;
#pragma unroll
                                    for (int h = 0; h < 4; ++h) rope_store8(a, row, head, page, off, i0 + 8 * h, av + 8 * h, bv + 8 * h, cr + 8 * h, sr + 8 * h);
                                }
                            }
                        }
                    }
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
            if (lane == 0) mbar_arrive(ring.acc_empty);
            u = uend;
        }
    }
}

StreamK make_streamk(float* ws, int N, int K, int bn, int G, int rows, bool fp8) {
    const int ke = fp8 ? 2 * BLOCK_K : BLOCK_K;
    StreamK sk{}; sk.ws = ws; sk.bn = bn; sk.rows = rows > 128 ? 256 : 128; sk.kb = (K + ke - 1) / ke; sk.n_tiles = (N + bn - 1) / bn;
    sk.total = (long long)sk.n_tiles * sk.kb; sk.G = (int)std::min<long long>(G, sk.total);
    sk.l2_prefetch_units = 0;
    return sk;
}
size_t streamk_ws_bytes(int N, int bn, int G, int rows) { return (size_t)(G + (N + bn - 1) / bn) * (rows > 128 ? 256 : 128) * bn * sizeof(float); }

template <int BN, int MT, int FUSE = 0>
static cudaError_t launch_sk(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, const StreamK& sk, cudaStream_t stream, SkFuse fz = SkFuse{}) {
    if (fz.w8.a) {
        // fp8: one row tile and N <= 128 only, and no fused SwiGLU.  With the promotion temporary, a second 64 x 128 fragment (MT = 2) or the
        // SwiGLU finisher's chunk buffers exceed the 168 registers per thread (ptxas spills); those shapes take the tile kernel / the consumer.
        if constexpr (BN <= 128 && MT == 1 && FUSE != 1)
            return launch_gemm_kernel<gemm_streamk_kernel<BN, MT, FUSE, true>>(dim3(sk.G), SkCfg<BN, MT, true>::SMEM_BYTES, stream, *tmA, *tmB, M, sk, fz);
        return cudaErrorInvalidValue;
    }
    return launch_gemm_kernel<gemm_streamk_kernel<BN, MT, FUSE>>(dim3(sk.G), SkCfg<BN, MT>::SMEM_BYTES, stream, *tmA, *tmB, M, sk, fz);
}
// fp8: both scale arrays or neither, K in whole 16-byte TMA rows
static bool w8_bad(const W8Scales& w8, int K) { return (w8.a == nullptr) != (w8.b == nullptr) || (w8.a && (K % 16) != 0); }
cudaError_t launch_gemm_streamk_swiglu(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int F, int K, const StreamK& sk, void* act,
                                       unsigned int* tile_flags, cudaStream_t stream, W8Scales w8) {
    if (M <= 0 || M > BLOCK_M || sk.rows != 128 || sk.bn != 128 || (F % 16) != 0 || (K % 8) != 0 || !act || !tile_flags || w8_bad(w8, K)) return cudaErrorInvalidValue;
    if (sk.G > sm_count_cached()) return cudaErrorInvalidValue;      // finishing CTAs wait for publishing CTAs: all must be resident
    SkFuse fz{}; fz.act = reinterpret_cast<uint16_t*>(act); fz.F = F; fz.tile_flags = tile_flags; fz.N = 2 * F; fz.w8 = w8;
    return launch_sk<128, 1, 1>(tmA, tmB, M, sk, stream, fz);
}
cudaError_t launch_gemm_streamk_resid(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, void* x, int ldx,
                                      unsigned int* tile_flags, cudaStream_t stream, W8Scales w8) {
    if (M <= 0 || M > BLOCK_M || sk.rows != 128 || sk.bn != 128 || (N % 32) != 0 || (K % 8) != 0 || !x || !tile_flags || (ldx % 8) != 0 || w8_bad(w8, K)) return cudaErrorInvalidValue;
    if (sk.G > sm_count_cached()) return cudaErrorInvalidValue;      // finishing CTAs wait for publishing CTAs: all must be resident
    SkFuse fz{}; fz.tile_flags = tile_flags; fz.x = reinterpret_cast<uint16_t*>(x); fz.ldx = ldx; fz.N = N; fz.w8 = w8;
    return launch_sk<128, 1, 2>(tmA, tmB, M, sk, stream, fz);
}
cudaError_t launch_gemm_streamk_rope(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, const SkRopeArgs& rope,
                                     unsigned int* tile_flags, cudaStream_t stream, W8Scales w8) {
    if (M <= 0 || M > BLOCK_M || sk.rows != 128 || sk.bn != 128 || (K % 8) != 0 || !tile_flags || w8_bad(w8, K)) return cudaErrorInvalidValue;
    if ((rope.D != 64 && rope.D != 128) || N != (rope.nh + 2 * rope.nkv) * rope.D) return cudaErrorInvalidValue;      // BN must be a multiple of D; chunks of 32 never straddle a head
    if (sk.G > sm_count_cached()) return cudaErrorInvalidValue;
    SkFuse fz{}; fz.tile_flags = tile_flags; fz.N = N; fz.rope = rope; fz.w8 = w8;
    return launch_sk<128, 1, 3>(tmA, tmB, M, sk, stream, fz);
}
cudaError_t launch_gemm_streamk(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const StreamK& sk, cudaStream_t stream, W8Scales w8) {
    if (M <= 0 || M > sk.rows || (N % 8) != 0 || (K % 8) != 0 || w8_bad(w8, K)) return cudaErrorInvalidValue;
    SkFuse fz{}; fz.N = N; fz.w8 = w8;
    if (sk.rows == 256) return sk.bn == 128 ? launch_sk<128, 2>(tmA, tmB, M, sk, stream, fz) : cudaErrorInvalidValue;
    if (sk.bn == 256) return launch_sk<256, 1>(tmA, tmB, M, sk, stream, fz);      // bf16 only
    if (sk.bn == 128) return launch_sk<128, 1>(tmA, tmB, M, sk, stream, fz);      // more CTAs than SMs run in waves: the plain kernel never waits on another CTA
    if (sk.bn == 64) return launch_sk<64, 1>(tmA, tmB, M, sk, stream, fz);       // half the partial bytes again; per-projection opt-in (sk_bn_o / sk_bn_down / sk_bn_qkv)
    return cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------
__global__ void argmax_reduce_kernel(const float* __restrict__ val, const int* __restrict__ idx, int M, int n_tiles,
                                     int32_t* __restrict__ out_ids, float* __restrict__ out_val) {
    const int row = blockIdx.x;
    griddep_launch(); griddep_wait();
    float bv; int bi;
    block_argmax_row(val, idx, row, n_tiles, bv, bi);
    if (threadIdx.x == 0) {
        out_ids[row] = bi == 0x7fffffff ? 0 : bi;
        if (out_val) out_val[row] = bv;
    }
}

cudaError_t launch_argmax_reduce(const float* amax_val, const int* amax_idx, int M, int n_tiles, int32_t* out_ids,
                                 float* out_val, cudaStream_t stream) {
    return launch_k(argmax_reduce_kernel, dim3(M), dim3(256), 0, stream, amax_val, amax_idx, M, n_tiles, out_ids, out_val);
}

}  // namespace oa
