// sk_consumers.cuh — the consumers of stream-K partials as device functions: each adds a tile's fp32 partials in CTA
// order (deterministic) and finishes the op with the bf16x8 epilogue helpers of common.cuh.  The stand-alone consumer kernels
// (elementwise.cu, tp_comm.cu) run these functions; the GEMM epilogues that finish an op themselves (gemm_wgmma.cu FUSE=1/2/3,
// gemm_clusterk.cu) sum in the same order and call the same helpers and kv_store8, so every path produces bit-identical results.
#pragma once
#include "common.cuh"
#include "kernels.hpp"

namespace oa {

OA_DEVINL void named_bar_sync(int id, int n_threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory"); }

// CTAs c_first..c_last own pieces of `tile` (sk_tile_ctas, kernels.hpp); their partials are added in that order.
OA_DEVINL void sk_sum8(const StreamK& sk, int row, int col, float (&acc)[8]) {
    const uint32_t tile = (uint32_t)col / (uint32_t)sk.bn, cc = (uint32_t)col - tile * (uint32_t)sk.bn;
    uint32_t c_first, c_last;
    sk_tile_ctas(sk, tile, c_first, c_last);
    const int n = (int)(c_last - c_first) + 1;
    const size_t slot_stride = (size_t)sk.rows * sk.bn;
    const float* p = sk.ws + ((size_t)(c_first + tile) * sk.rows + row) * sk.bn + cc;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    // issue up to 6 partials' loads back to back (independent L2 round trips), then add them in CTA order
    for (int i = 0; i < n; i += 6) {
        float4 a[6], b[6];
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            if (i + j < n) {
                const float4* q4 = reinterpret_cast<const float4*>(p + (size_t)(i + j) * slot_stride);
                a[j] = __ldcg(q4); b[j] = __ldcg(q4 + 1);
            } else { a[j] = make_float4(0.f, 0.f, 0.f, 0.f); b[j] = a[j]; }
        }
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            if (i + j < n) {
                acc[0] += a[j].x; acc[1] += a[j].y; acc[2] += a[j].z; acc[3] += a[j].w;
                acc[4] += b[j].x; acc[5] += b[j].y; acc[6] += b[j].z; acc[7] += b[j].w;
            }
        }
    }
}

// Two 8-column groups of the SAME tile (a RoPE pair: columns c and c + D/2): one index computation, both groups' partial loads in
// flight together, each summed in CTA order exactly as sk_sum8 does.
OA_DEVINL void sk_sum8_pair(const StreamK& sk, int row, int col_a, int col_b, float (&acc_a)[8], float (&acc_b)[8]) {
    const uint32_t tile = (uint32_t)col_a / (uint32_t)sk.bn;
    if ((uint32_t)col_b / (uint32_t)sk.bn != tile) { sk_sum8(sk, row, col_a, acc_a); sk_sum8(sk, row, col_b, acc_b); return; }
    const uint32_t ca = (uint32_t)col_a - tile * (uint32_t)sk.bn, cb = (uint32_t)col_b - tile * (uint32_t)sk.bn;
    uint32_t c_first, c_last;
    sk_tile_ctas(sk, tile, c_first, c_last);
    const int n = (int)(c_last - c_first) + 1;
    const size_t slot_stride = (size_t)sk.rows * sk.bn;
    const float* p = sk.ws + ((size_t)(c_first + tile) * sk.rows + row) * sk.bn;
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc_a[i] = 0.f; acc_b[i] = 0.f; }
    for (int i = 0; i < n; i += 4) {
        float4 a0[4], a1[4], b0[4], b1[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (i + j < n) {
                const float* q = p + (size_t)(i + j) * slot_stride;
                a0[j] = __ldcg(reinterpret_cast<const float4*>(q + ca)); a1[j] = __ldcg(reinterpret_cast<const float4*>(q + ca) + 1);
                b0[j] = __ldcg(reinterpret_cast<const float4*>(q + cb)); b1[j] = __ldcg(reinterpret_cast<const float4*>(q + cb) + 1);
            } else { a0[j] = make_float4(0.f, 0.f, 0.f, 0.f); a1[j] = a0[j]; b0[j] = a0[j]; b1[j] = a0[j]; }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (i + j < n) {
                acc_a[0] += a0[j].x; acc_a[1] += a0[j].y; acc_a[2] += a0[j].z; acc_a[3] += a0[j].w;
                acc_a[4] += a1[j].x; acc_a[5] += a1[j].y; acc_a[6] += a1[j].z; acc_a[7] += a1[j].w;
                acc_b[0] += b0[j].x; acc_b[1] += b0[j].y; acc_b[2] += b0[j].z; acc_b[3] += b0[j].w;
                acc_b[4] += b1[j].x; acc_b[5] += b1[j].y; acc_b[6] += b1[j].z; acc_b[7] += b1[j].w;
            }
        }
    }
}

// x[t,:] += sum of partials (bf16 residual stream), y[t,:] = rmsnorm(x[t,:]) * g.  SK_RESID_THREADS threads (tid) per row, so that
// at H <= 4096 every thread owns ONE 16-byte item and all its partial loads are in flight together; `red` = 16 floats of
// shared memory, `bar_id` = a hardware barrier those threads own.
constexpr int SK_RESID_THREADS = 512;
template <int VPT, bool SUM = true>     // SUM == false: the residual stream already holds x + projection (fused GEMM epilogue); only normalise
OA_DEVINL void sk_resid_rmsnorm_row(const StreamK& sk, int t, int tid, float* red, int bar_id, uint4* __restrict__ x,
                                    const uint4* __restrict__ g, uint4* __restrict__ y, int H8, float inv_h, float eps) {
    uint4* xr = x + (size_t)t * H8;
    uint4 v[VPT], gg[VPT];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
        const int i = tid + k * SK_RESID_THREADS;
        if (i < H8) {
            const uint4 xo = __ldcg(xr + i);
            gg[k] = g[i];                              // needed only after the reduction: its latency hides behind the partial loads
            uint4 xn = xo;
            if constexpr (SUM) {
                float acc[8];
                sk_sum8(sk, t, i * 8, acc);
                add_bf16x8(acc, xo);
                xn = pack_bf16x8(acc);
                xr[i] = xn;
            }
            v[k] = xn;
            ss = sumsq_bf16x8(xn, ss);
        }
    }
    ss = warp_sum(ss);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    named_bar_sync(bar_id, SK_RESID_THREADS);
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < SK_RESID_THREADS / 32; ++w) tot += red[w];
    const float r = 1.0f / sqrtf(tot * inv_h + eps);
    uint4* yr = y + (size_t)t * H8;
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
        const int i = tid + k * SK_RESID_THREADS;
        if (i < H8) yr[i] = rms_scale_bf16x8(v[k], r, gg[k]);
    }
}

// act[t, i*8 .. i*8+8) = silu(gate) * up.  Physical columns of the fused gate/up GEMM: per 32-column block, 16 gate then 16 up.
OA_DEVINL void sk_swiglu_item(const StreamK& sk, int t, int i, uint4* __restrict__ act, int F8) {
    const int f0 = i * 8, blk = f0 >> 4, o = f0 & 15;
    float gt[8], up[8];
    sk_sum8(sk, t, blk * 32 + o, gt);
    sk_sum8(sk, t, blk * 32 + 16 + o, up);
    act[(size_t)t * F8 + i] = swiglu_bf16x8(gt, up);
}

// summed qkv columns [col, col + 8) + bias, then rounded: the projection output is a bf16 tensor
OA_DEVINL void qkv_finish8(const uint16_t* bias, int col, float* v) {
    if (bias) add_bf16x8(v, *reinterpret_cast<const uint4*>(bias + col));
    round_bf16x8(v);
}

// destination row of q / k / v head `head` (in qkv column order) of token row t: q_out, or the paged K / V plane at (page, off)
OA_DEVINL uint16_t* rope_dst_row(const SkRopeArgs& a, int t, int head, int page, int off) {
    if (head < a.nh) return a.q_out + (size_t)t * a.nh * a.D + (size_t)head * a.D;
    if (head < a.nh + a.nkv) return kv_row(a.kv_base, a.k_plane_row0, page, a.nkv, head - a.nh, a.page_size, off, a.D);
    return kv_row(a.kv_base, a.v_plane_row0, page, a.nkv, head - a.nh - a.nkv, a.page_size, off, a.D);
}

// Stores 8 finished bf16 lanes (columns i0..i0+7 of head `head`) where rope_dst_row points: q_out, or the paged K / V plane.  Every
// writer of the KV cache stores through here.  fp8 cache: byte = e4m3(bf16 value * inv_scale); K as [token][D] (8 consecutive bytes), V
// transposed inside its (page, kv head) block as [D][page_size] (8 bytes page_size apart).
OA_DEVINL void kv_store8(const SkRopeArgs& a, int t, int head, int page, int off, int i0, uint4 v) {
    if (!a.kv_fp8 || head < a.nh) { *reinterpret_cast<uint4*>(rope_dst_row(a, t, head, page, off) + i0) = v; return; }
    float f[8];
    unpack_bf16x8(v, f);
    uint8_t* base = reinterpret_cast<uint8_t*>(a.kv_base);
    if (head < a.nh + a.nkv) {
        *reinterpret_cast<uint2*>(base + (size_t)(a.k_plane_row0 + ((int64_t)page * a.nkv + head - a.nh) * a.page_size + off) * a.D + i0) =
            pack_e4m3x8(f, a.k_inv_scale);
        return;
    }
    const uint2 b = pack_e4m3x8(f, a.v_inv_scale);
    uint8_t* col = base + (size_t)(a.v_plane_row0 + ((int64_t)page * a.nkv + head - a.nh - a.nkv) * a.page_size) * a.D + (size_t)i0 * a.page_size + off;
#pragma unroll
    for (int k = 0; k < 8; ++k) col[(size_t)k * a.page_size] = (uint8_t)(((k < 4 ? b.x : b.y) >> (8 * (k & 3))) & 0xff);
}
// RoPE of 8 (lo, hi) pairs of head `head` (columns i0.. and i0 + D/2..) and the store of both halves
OA_DEVINL void rope_store8(const SkRopeArgs& a, int t, int head, int page, int off, int i0, const float* lo, const float* hi, const float* cs, const float* sn) {
    uint4 ra, rb;
    rope_bf16x8(lo, hi, cs, sn, ra, rb);
    kv_store8(a, t, head, page, off, i0, ra);
    kv_store8(a, t, head, page, off, i0 + (a.D >> 1), rb);
}

OA_DEVINL int sk_rope_items_per_row(const SkRopeArgs& a) { return (a.nh + a.nkv) * (a.D >> 4) + a.nkv * (a.D >> 3); }
// item w of token row t: w < (nh+nkv)*D/16 rotates 8 (lo, hi) pairs of one q or k head; the rest copy 8 elements of v
OA_DEVINL void sk_rope_item(const StreamK& sk, const SkRopeArgs& a, int t, int w) {
    const int D = a.D, half = D >> 1, vec_per_head = half >> 3;
    const int slot = a.slots[t];
    const int page = slot / a.page_size, off = slot - page * a.page_size;
    const int n_rot = (a.nh + a.nkv) * vec_per_head;
    if (w < n_rot) {
        const int pos = a.positions[t];
        const int head = w / vec_per_head, i0 = (w - head * vec_per_head) * 8;
        float av[8], bv[8];
        sk_sum8_pair(sk, t, head * D + i0, head * D + i0 + half, av, bv);
        qkv_finish8(a.bias, head * D + i0, av);
        qkv_finish8(a.bias, head * D + i0 + half, bv);
        rope_store8(a, t, head, page, off, i0, av, bv, a.rope_cos + (size_t)pos * half + i0, a.rope_sin + (size_t)pos * half + i0);
    } else {
        const int wv = w - n_rot;
        const int head = a.nh + a.nkv + wv / (D >> 3), i0 = (wv % (D >> 3)) * 8;
        float vv[8];
        sk_sum8(sk, t, head * D + i0, vv);
        qkv_finish8(a.bias, head * D + i0, vv);
        kv_store8(a, t, head, page, off, i0, pack_bf16x8(vv));
    }
}

}  // namespace oa
