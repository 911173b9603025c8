// gemm_pipe.cuh — the warp-specialised pipeline every GEMM kernel (gemm_wgmma.cu, gemm_clusterk.cu) is built on:
//   warp 8    : TMA producer — per unit (one 64-wide k-block of one output tile) MT boxes {64 x 128} of A and one {64 x BN} of B into
//               a STAGES-deep shared-memory ring (128-byte swizzle), completion on `full` mbarriers;
//   warps 0-7 : two consumer warpgroups; warpgroup g issues wgmma 64 x BN x 16 (bf16 -> fp32 in registers) for rows [64g, 64g + 64) of
//               each 128-row A tile and releases ring slots (`empty`) as their MMAs retire.
// fp8 (e4m3) operands (RingCfg FP8): the same bytes per unit hold 128 K elements; wgmma 64 x BN x 32, promoted to fp32 per unit.
// Shared memory: [ring][accumulator region][barriers], 1024-byte aligned (the 128-byte swizzle atom).
#pragma once
#include "common.cuh"
#include "kernels.hpp"

namespace oa {

static constexpr int BLOCK_M = 128;
static constexpr int BLOCK_K = 64;     // 64 bf16 = 128 B = one swizzle row
static constexpr int EPI_WARP0 = 0, PRODUCER_WARP = 8, CONSUMER_WARPS = 8;
// 2 consumer warpgroups + 1 producer warp: 9 warps leave 168 registers per thread, room for a 64 x 256 fp32 fragment (128)
static constexpr int GEMM_THREADS = 32 * (PRODUCER_WARP + 1);
#define OA_GEMM_REGS __launch_bounds__(GEMM_THREADS, 1)
static constexpr int RASTER_GROUP_M = 16;
static constexpr int SMEM_LIMIT = 232448;                           // opt-in shared memory of one CTA on sm_90
static constexpr int RING_SLACK = 1024 /*align*/ + 256 /*barriers*/;

// ring of STAGES units (MT A tiles + one B tile each) next to an accumulator region of ACC bytes (default: the fp32 tile [MT * 128][BN]).
// A unit is one 128-byte swizzle row of K: 64 bf16 elements, or 128 e4m3 elements when FP8 (same bytes, same ring geometry).
template <int BN_, int MT_, int STAGES_, int ACC = MT_ * BLOCK_M * BN_ * 4, bool FP8_ = false>
struct RingCfg {
    static constexpr int BN = BN_, MT = MT_, STAGES = STAGES_;
    static constexpr bool FP8 = FP8_;
    static constexpr int KE = FP8 ? 2 * BLOCK_K : BLOCK_K;        // K elements per unit
    static constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;        // 16 KB
    static constexpr int A_BYTES = MT * A_TILE_BYTES;
    static constexpr int B_BYTES = BN * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int ACC_BYTES = ACC;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + RING_SLACK;
    static_assert(STAGES >= 2 && SMEM_BYTES <= SMEM_LIMIT, "shared memory budget of one CTA");
};
// the deepest ring, at most `cap` stages, that fits next to the fp32 accumulator tile
constexpr int ring_stages_fit(int bn, int mt, int cap) {
    const int fit = (SMEM_LIMIT - mt * BLOCK_M * bn * 4 - RING_SLACK) / (mt * BLOCK_M * BLOCK_K * 2 + bn * BLOCK_K * 2);
    return fit < cap ? fit : cap;
}

struct Ring {
    uint8_t* smem;                     // stage s at smem + s * STAGE_BYTES: A tiles, then the B tile
    float* acc;                        // accumulator region
    uint64_t* full_bar;                // [STAGES]
    uint64_t* empty_bar;               // [STAGES], one arrival per consumer warp
    uint64_t* acc_full;                // one arrival per consumer warp: the accumulator region holds a tile
    uint64_t* acc_empty;               // one arrival per epilogue warp: the epilogue has drained it
};
// Carve the ring out of dynamic shared memory, initialise its barriers and prefetch the tensor maps; then let the next kernel launch.
template <class Cfg>
OA_DEVINL Ring ring_setup(uint8_t* smem_raw, const CUtensorMap* tmA, const CUtensorMap* tmB) {
    Ring r;
    r.smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    r.acc = reinterpret_cast<float*>(r.smem + Cfg::STAGES * Cfg::STAGE_BYTES);
    r.full_bar = reinterpret_cast<uint64_t*>(r.smem + Cfg::STAGES * Cfg::STAGE_BYTES + Cfg::ACC_BYTES);
    r.empty_bar = r.full_bar + Cfg::STAGES;
    r.acc_full = r.empty_bar + Cfg::STAGES;
    r.acc_empty = r.acc_full + 1;
    if (threadIdx.x == PRODUCER_WARP * 32) {
        tma_prefetch_desc(tmA); tma_prefetch_desc(tmB);
        for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&r.full_bar[s], 1); mbar_init(&r.empty_bar[s], CONSUMER_WARPS); }
        mbar_init(r.acc_full, CONSUMER_WARPS); mbar_init(r.acc_empty, 4);
        fence_barrier_init();
    }
    __syncthreads();
    griddep_launch();
    return r;
}

// Producer (one thread): units [0, n) in order; unit(i, kx, a_row, b_row) gives the k coordinate of unit i and the first rows of its A
// tiles and its B tile.  WEIGHTS_FIRST: B is written by no kernel of the chain, so the first STAGES units' B tiles are issued — and the
// next l2_prefetch units' B boxes pulled into L2 — before griddepcontrol.wait, while the predecessor still runs; `unit` must then be a
// function of i alone (those units are visited more than once).  Otherwise it is called exactly once per unit, in increasing i.
template <class Cfg, bool WEIGHTS_FIRST, class Unit>
OA_DEVINL void ring_produce(const Ring& r, const CUtensorMap* tmA, const CUtensorMap* tmB, int n, Unit unit, uint64_t a_policy,
                            uint64_t b_policy, int l2_prefetch = 0) {
    auto load_a = [&](int slot, int kx, int a_row) {
#pragma unroll
        for (int m = 0; m < Cfg::MT; ++m)
            tma_load_2d(r.smem + slot * Cfg::STAGE_BYTES + m * Cfg::A_TILE_BYTES, tmA, &r.full_bar[slot], kx, a_row + m * BLOCK_M, a_policy);
    };
    int pre = 0;
    if constexpr (WEIGHTS_FIRST) {
        pre = n < Cfg::STAGES ? n : Cfg::STAGES;
        for (int i = 0; i < pre; ++i) {
            int kx, a_row, b_row; unit(i, kx, a_row, b_row);
            mbar_expect_tx(&r.full_bar[i], Cfg::STAGE_BYTES);
            tma_load_2d(r.smem + i * Cfg::STAGE_BYTES + Cfg::A_BYTES, tmB, &r.full_bar[i], kx, b_row, b_policy);
        }
        const int pf_end = pre + l2_prefetch < n ? pre + l2_prefetch : n;
        for (int i = pre; i < pf_end; ++i) { int kx, a_row, b_row; unit(i, kx, a_row, b_row); tma_prefetch_l2_2d(tmB, kx, b_row); }
    }
    griddep_wait();
    for (int i = 0; i < pre; ++i) { int kx, a_row, b_row; unit(i, kx, a_row, b_row); load_a(i, kx, a_row); }
    int s = pre == Cfg::STAGES ? 0 : pre; uint32_t ph = pre == Cfg::STAGES ? 1 : 0;
    for (int i = pre; i < n; ++i) {
        int kx, a_row, b_row; unit(i, kx, a_row, b_row);
        mbar_wait(&r.empty_bar[s], ph ^ 1);
        mbar_expect_tx(&r.full_bar[s], Cfg::STAGE_BYTES);
        load_a(s, kx, a_row);
        tma_load_2d(r.smem + s * Cfg::STAGE_BYTES + Cfg::A_BYTES, tmB, &r.full_bar[s], kx, b_row, b_policy);
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
    }
}

template <class Cfg>
OA_DEVINL void wg_mma_run_e4m3(float (&d)[Cfg::MT][Cfg::BN / 2], const Ring& r, int& s, uint32_t& ph, int n_kb);
// Consumer side of the ring: n_kb units into this warpgroup's registers (rows [64g, 64g + 64) of each of the MT 128-row A tiles).
// One wgmma group stays in flight; a slot is released (one arrival per consumer warp) once the group that read it has retired.
template <class Cfg>
OA_DEVINL void wg_mma_run(float (&d)[Cfg::MT][Cfg::BN / 2], const Ring& r, int& s, uint32_t& ph, int n_kb) {
    if constexpr (Cfg::FP8) { wg_mma_run_e4m3<Cfg>(d, r, s, ph, n_kb); return; }
    constexpr int BN = Cfg::BN;
    const uint32_t g_off = (threadIdx.x >> 7) * 64 * 128;
    const bool leader = (threadIdx.x & 31) == 0;
    int prev = -1;
    for (int i = 0; i < n_kb; ++i) {
        mbar_wait(&r.full_bar[s], ph);
        const uint32_t st = smem_u32(r.smem) + (uint32_t)(s * Cfg::STAGE_BYTES);
        const uint64_t db = gmma_desc_sw128(st + (uint32_t)Cfg::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int m = 0; m < Cfg::MT; ++m) {
            const uint64_t da = gmma_desc_sw128(st + (uint32_t)(m * Cfg::A_TILE_BYTES) + g_off);
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
        if (prev >= 0 && leader) mbar_arrive(&r.empty_bar[prev]);
        prev = s;
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && leader) mbar_arrive(&r.empty_bar[prev]);
}
// e4m3 operands: a unit is 128 K elements, four k32 wgmmas per 128-column half.  They go into a zero-initialised fragment that is then
// added to d in fp32 registers ("promotion": the fp8 tensor-core accumulator keeps only about 14 mantissa bits, so a long K is never summed
// there).  Each group is retired before its sum is promoted, so its slot is released at once; the producer keeps the ring full meanwhile.
// The temporary is 64 columns wide (32 registers): a 64 x 128 one leaves the fused finishers too few registers.
template <class Cfg>
OA_DEVINL void wg_mma_run_e4m3(float (&d)[Cfg::MT][Cfg::BN / 2], const Ring& r, int& s, uint32_t& ph, int n_kb) {
    constexpr int BN = Cfg::BN, NW = BN > 64 ? 64 : BN;
    const uint32_t g_off = (threadIdx.x >> 7) * 64 * 128;
    const bool leader = (threadIdx.x & 31) == 0;
    for (int i = 0; i < n_kb; ++i) {
        mbar_wait(&r.full_bar[s], ph);
        const uint32_t st = smem_u32(r.smem) + (uint32_t)(s * Cfg::STAGE_BYTES);
        const uint64_t db = gmma_desc_sw128(st + (uint32_t)Cfg::A_BYTES);
#pragma unroll
        for (int m = 0; m < Cfg::MT; ++m) {
            const uint64_t da = gmma_desc_sw128(st + (uint32_t)(m * Cfg::A_TILE_BYTES) + g_off);
#pragma unroll
            for (int nb = 0; nb < BN / NW; ++nb) {
                float t[NW / 2] = {};
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_e4m3<NW>(t, da + (uint64_t)(k * 2), db + (uint64_t)(nb * NW * 8 + k * 2), k > 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<0>();
#pragma unroll
                for (int j = 0; j < NW / 2; ++j) d[m][nb * (NW / 2) + j] += t[j];
            }
        }
        if (leader) mbar_arrive(&r.empty_bar[s]);
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
    }
}
// fp8: d[row][col] *= s_a[row] * s_b[col], rows from row0 (the first of the MT 128-row tiles), columns from col0; rows >= M and columns
// >= N get 0 (their TMA boxes were zero-filled).  s_a is written by the quantiser that precedes the GEMM, hence the dependency wait.
template <int BN, int MT>
OA_DEVINL void wg_scale_frag(float (&d)[MT][BN / 2], const W8Scales& w8, int row0, int col0, int M, int N) {
    griddep_wait();
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3, g = threadIdx.x >> 7;
#pragma unroll
    for (int m = 0; m < MT; ++m) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = row0 + m * BLOCK_M + g * 64 + 16 * w + (lane >> 2) + 8 * h;
            const float sa = row < M ? __ldg(w8.a + row) : 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = col0 + 8 * j + 2 * (lane & 3);          // even, and N % 8 == 0: both columns or neither are in range
                const float2 sb = col < N ? __ldg(reinterpret_cast<const float2*>(w8.b + col)) : make_float2(0.f, 0.f);
                d[m][4 * j + 2 * h] *= sa * sb.x;
                d[m][4 * j + 2 * h + 1] *= sa * sb.y;
                if ((j & 3) == 3) asm volatile("" ::: "memory");       // four loads in flight at a time: the scales never compete with d for registers
            }
        }
    }
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

// Grouped rasterisation: tiles walk bands of RASTER_GROUP_M row tiles, M fastest inside a band, so a band of A (16 x 128 rows) stays
// L2-resident while each B tile is streamed from HBM once per band instead of once per row tile.
OA_DEVINL void raster_tile(int idx, int m_tiles, int n_tiles, int& m_blk, int& n_blk) {
    const int per_band = RASTER_GROUP_M * n_tiles;
    const int band = idx / per_band, within = idx - band * per_band;
    const int m0 = band * RASTER_GROUP_M;
    const int rows = (m_tiles - m0) < RASTER_GROUP_M ? (m_tiles - m0) : RASTER_GROUP_M;
    m_blk = m0 + within % rows; n_blk = within / rows;
}

// Launch one GEMM kernel of GEMM_THREADS threads, raising its dynamic shared-memory limit first (once per device).
template <auto KERN, class... Args>
static cudaError_t launch_gemm_kernel(LaunchGrid grid, int smem, cudaStream_t stream, const Args&... args) {
    static bool attr_done[16] = {};
    if (cudaError_t e = ensure_dynamic_smem(KERN, smem, attr_done); e != cudaSuccess) return e;
    return launch_k(KERN, grid, dim3(GEMM_THREADS), smem, stream, args...);
}

}  // namespace oa
