// gemm_clusterk.cu — decode projections with FEW output tiles (o, down, qkv: 32-48 tiles of 128 columns on 132 SMs) as a
// cluster split-K GEMM: the S CTAs of one thread-block cluster own ONE 128 x 128 output tile and a 1/S slice of K each, reduce their
// register accumulators through distributed shared memory and finish the epilogue together — no fp32 partial round trip through L2, no
// consumer launch, no serial tail of a few finishing CTAs (the weakness of the stream-K finisher fusion on these shapes).
//
//   grid = n_tiles x S CTAs, cluster (S,1,1); CTA (tile, r) streams k-blocks [r*kb/S, (r+1)*kb/S) of the tile's weights
//   warp 8   : TMA producer (weights issued BEFORE griddepcontrol.wait: they depend on no predecessor)
//   warps 0-7: two warpgroups, wgmma 64 x 128 x 16 each (rows [64g, 64g + 64)) into registers, then st.shared::cluster of the fragments
//              into the OWNER CTA of each 32 x 64 "pair unit" (8 per tile, owner = unit % S);
//              after one cluster barrier every CTA sums the S partials of its own units IN RANK ORDER (deterministic) and applies the
//              epilogue with warps 0-3: residual add into the bf16 stream (o / down) or bias + RoPE + paged-KV write (qkv).
// A pair unit = rows [32q, 32q+32) x the two 32-column chunks that RoPE rotates together (columns i and i + D/2 of one head), so every
// epilogue is thread-local.  The K split differs from the stream-K path, so results are equal to it only up to fp32 summation order
// (parity against the oracle holds with the same tolerance; the bit-identity test covers the stream-K variants among themselves).
#include <algorithm>

#include "gemm_pipe.cuh"
#include "sk_consumers.cuh"

namespace oa {

static constexpr int CK_BN = 128;
static constexpr int CK_ROW_F = 36;                              // 32 + 4 pad floats: conflict-free 16-byte accesses
static constexpr int CK_BUF_F = 32 * CK_ROW_F;                   // one 32 x 32 partial chunk
template <int S> constexpr int CK_SLOTS = (8 + S - 1) / S;      // pair units a CTA may own
// the accumulator region is the receive buffer [SLOTS][2 members][S partials][32][36]
template <int S> using CkCfg = RingCfg<CK_BN, 1, 4, CK_SLOTS<S> * 2 * S * CK_BUF_F * 4>;

struct CkEpi {
    int kind;                           // 2: x[M, ldx] += acc (residual stream, bf16, in place)   3: bias + RoPE + paged-KV write
    uint16_t* x; int ldx; int N;
    SkRopeArgs rope;
};

OA_DEVINL uint32_t ck_cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
OA_DEVINL uint32_t ck_mapa(uint32_t addr, uint32_t rank) { uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r; }
OA_DEVINL void ck_st_cluster_f2(uint32_t addr, float a, float b) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
OA_DEVINL void ck_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// chunk c (32 columns) of a tile -> (pair index within the row block, member 0 = low half / 1 = high half of the rotation)
template <int D> OA_DEVINL void ck_pair_of(int c, int& pidx, int& member) { if (D == 128) { pidx = c & 1; member = c >> 1; } else { pidx = c >> 1; member = c & 1; } }
template <int D> OA_DEVINL int ck_chunk_of(int pidx, int member) { return D == 128 ? pidx + 2 * member : 2 * pidx + member; }

template <int S, int D>
__global__ void OA_GEMM_REGS gemm_clusterk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                                  const int M, const int K, const CkEpi ep) {
    using Cfg = CkCfg<S>;
    constexpr int SLOTS = CK_SLOTS<S>;
    extern __shared__ uint8_t smem_raw[];
    const Ring ring = ring_setup<Cfg>(smem_raw, &tmA, &tmB);
    float* recv = ring.acc;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t rank = ck_cluster_rank();
    const int tile = (int)blockIdx.x / S;
    const int kb_total = (K + BLOCK_K - 1) / BLOCK_K;
    const int kb0 = (int)((long long)rank * kb_total / S), kb1 = (int)((long long)(rank + 1) * kb_total / S), n_kb = kb1 - kb0;   // kb_total >= S (the launchers refuse less)

    float d[1][CK_BN / 2] = {};
    if (warp == PRODUCER_WARP) {
        if (lane == 0) {
            auto unit = [&](int i, int& kx, int& a_row, int& b_row) { kx = (kb0 + i) * BLOCK_K; a_row = 0; b_row = tile * CK_BN; };
            ring_produce<Cfg, true>(ring, &tmA, &tmB, n_kb, unit, kEvictLast, kEvictFirst);
        }
    } else if (warp < CONSUMER_WARPS) {
        int s = 0; uint32_t ph = 0;
        wg_mma_run<Cfg>(d, ring, s, ph, n_kb);
    }
    // every CTA of the cluster is running (co-scheduled) and past its setup before anybody writes into a peer's shared memory
    ck_cluster_sync();
    if (warp < CONSUMER_WARPS) {
        // fragment (row, col pair) -> the pair unit that owns it, in the owner CTA's receive buffer
        griddep_wait();
        const int g = warp >> 2, w = warp & 3;
        const uint32_t recv_base = smem_u32(recv);
#pragma unroll
        for (int j = 0; j < CK_BN / 8; ++j) {
            int pidx, member; ck_pair_of<D>(j >> 2, pidx, member);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = g * 64 + 16 * w + (lane >> 2) + 8 * h, col = 8 * j + 2 * (lane & 3);
                const int pu = (row >> 5) * 2 + pidx, owner = pu % S, slot = pu / S;
                const uint32_t local = recv_base + (uint32_t)((((slot * 2 + member) * S + (int)rank) * CK_BUF_F + (row & 31) * CK_ROW_F + (col & 31)) * 4);
                ck_st_cluster_f2(ck_mapa(local, (uint32_t)owner), d[0][4 * j + 2 * h], d[0][4 * j + 2 * h + 1]);
            }
        }
    }
    ck_cluster_sync();                                            // all partials of my units have landed in my shared memory
    if (warp < 4) {
        const int t = (int)threadIdx.x;                           // 0..127
        const int r32 = t >> 2, col8 = (t & 3) * 8;
#pragma unroll 1
        for (int slot = 0; slot < SLOTS; ++slot) {
            const int pu = (int)rank + slot * S;
            if (pu >= 8) break;
            const int q = pu >> 1, pidx = pu & 1;
            const int row = q * 32 + r32;
            float acc[2][8];
#pragma unroll
            for (int m = 0; m < 2; ++m) {
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[m][i] = 0.f;
#pragma unroll
                for (int p = 0; p < S; ++p) {                     // cluster-rank order = ascending k: a fixed order
                    const float* b = recv + ((slot * 2 + m) * S + p) * CK_BUF_F + r32 * CK_ROW_F + col8;
                    const float4 u0 = *reinterpret_cast<const float4*>(b), u1 = *reinterpret_cast<const float4*>(b + 4);
                    acc[m][0] += u0.x; acc[m][1] += u0.y; acc[m][2] += u0.z; acc[m][3] += u0.w;
                    acc[m][4] += u1.x; acc[m][5] += u1.y; acc[m][6] += u1.z; acc[m][7] += u1.w;
                }
            }
            if (row >= M) continue;
            const int col_lo = tile * CK_BN + ck_chunk_of<D>(pidx, 0) * 32 + col8, col_hi = tile * CK_BN + ck_chunk_of<D>(pidx, 1) * 32 + col8;
            if (ep.kind == 2) {
#pragma unroll
                for (int m = 0; m < 2; ++m) {
                    const int col = m ? col_hi : col_lo;
                    if (col >= ep.N) continue;
                    uint4* xp = reinterpret_cast<uint4*>(ep.x + (size_t)row * ep.ldx + col);
                    add_bf16x8(acc[m], *xp);
                    *xp = pack_bf16x8(acc[m]);
                }
            } else {
                if (col_lo >= ep.N) continue;
                const SkRopeArgs& a = ep.rope;
                const int half = D >> 1, head = col_lo / D, i0 = col_lo - head * D;          // i0 in [0, D/2): the low half of a rotation pair
                const int slot_tok = a.slots[row], page = slot_tok / a.page_size, off = slot_tok - page * a.page_size;
                qkv_finish8(a.bias, col_lo, acc[0]);
                qkv_finish8(a.bias, col_hi, acc[1]);
                if (head >= a.nh + a.nkv) {                       // V: straight copy of both halves into the V plane
                    kv_store8(a, row, head, page, off, i0, pack_bf16x8(acc[0]));
                    kv_store8(a, row, head, page, off, i0 + half, pack_bf16x8(acc[1]));
                } else {
                    const int pos = a.positions[row];
                    rope_store8(a, row, head, page, off, i0, acc[0], acc[1], a.rope_cos + (size_t)pos * half + i0, a.rope_sin + (size_t)pos * half + i0);
                }
            }
        }
    }
}

template <int S, int D>
static cudaError_t launch_ck(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const CkEpi& ep, cudaStream_t stream) {
    const int n_tiles = (N + CK_BN - 1) / CK_BN;
    return launch_gemm_kernel<gemm_clusterk_kernel<S, D>>(LaunchGrid(dim3(n_tiles * S), S), CkCfg<S>::SMEM_BYTES, stream, *tmA, *tmB, M, K, ep);
}

template <int D>
static cudaError_t launch_ck_s(int S, const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, const CkEpi& ep, cudaStream_t st) {
    switch (S) {
        case 2: return launch_ck<2, D>(tmA, tmB, M, N, K, ep, st);
        case 3: return launch_ck<3, D>(tmA, tmB, M, N, K, ep, st);
        case 4: return launch_ck<4, D>(tmA, tmB, M, N, K, ep, st);
        case 8: return launch_ck<8, D>(tmA, tmB, M, N, K, ep, st);
    }
    return cudaErrorInvalidValue;
}

// cluster size for an N x K projection on `sms` SMs: the largest of {8, 4, 3, 2} with n_tiles * S <= sms and >= 2 k-blocks per CTA
// (0: not worth it — fewer than min_fill_pct % of the SMs would stream)
int clusterk_pick(int N, int K, int sms, int min_fill_pct) {
    const int n_tiles = (N + CK_BN - 1) / CK_BN, kb = (K + BLOCK_K - 1) / BLOCK_K;
    for (int S : {8, 4, 3, 2})
        if (n_tiles * S <= sms && kb >= 2 * S) return (n_tiles * S * 100 >= sms * min_fill_pct) ? S : 0;
    return 0;
}

// every CTA of a cluster must own at least one k-block (the kernel's kb_total >= S)
static bool ck_too_short(int K, int S) { return (K + BLOCK_K - 1) / BLOCK_K < S; }

cudaError_t launch_gemm_clusterk_resid(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int S, void* x, int ldx, cudaStream_t stream) {
    if (M <= 0 || M > BLOCK_M || (N % 8) != 0 || (K % 8) != 0 || !x || (ldx % 8) != 0 || ck_too_short(K, S)) return cudaErrorInvalidValue;
    CkEpi ep{}; ep.kind = 2; ep.x = reinterpret_cast<uint16_t*>(x); ep.ldx = ldx; ep.N = N;
    return launch_ck_s<128>(S, tmA, tmB, M, N, K, ep, stream);          // D only fixes the unit pairing: any pairing suits the residual epilogue
}
cudaError_t launch_gemm_clusterk_rope(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int S, const SkRopeArgs& rope, cudaStream_t stream) {
    if (M <= 0 || M > BLOCK_M || (K % 8) != 0 || N != (rope.nh + 2 * rope.nkv) * rope.D || ck_too_short(K, S)) return cudaErrorInvalidValue;
    CkEpi ep{}; ep.kind = 3; ep.N = N; ep.rope = rope;
    if (rope.D == 128) return launch_ck_s<128>(S, tmA, tmB, M, N, K, ep, stream);
    if (rope.D == 64) return launch_ck_s<64>(S, tmA, tmB, M, N, K, ep, stream);
    return cudaErrorInvalidValue;
}

}  // namespace oa
