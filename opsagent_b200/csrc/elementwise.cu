// elementwise.cu — the HBM-bound glue kernels of the decode path: embedding gather, RMSNorm, row gather,
// RoPE + paged-KV write.  All use 16-byte vector accesses; one CTA per token row.
#include "common.cuh"
#include "kernels.hpp"
#include "sk_consumers.cuh"

namespace oa {

// out[t,:] = table[ids[t],:]   (ids outside [0,vocab) read row 0, as the oracle does)
__global__ void embed_gather_kernel(const int32_t* __restrict__ ids, const uint4* __restrict__ table, uint4* __restrict__ out,
                                    int H8, int vocab) {
    griddep_launch(); griddep_wait();
    const int t = blockIdx.x;
    int id = ids[t];
    if (id < 0 || id >= vocab) id = 0;
    const uint4* src = table + (size_t)id * H8;
    uint4* dst = out + (size_t)t * H8;
    for (int i = threadIdx.x; i < H8; i += blockDim.x) dst[i] = src[i];
}
cudaError_t launch_embed_gather(const int32_t* ids, const void* table, void* out, int T, int H, int vocab, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    return launch_k(embed_gather_kernel, dim3(T), dim3(128), 0, s, ids, reinterpret_cast<const uint4*>(table), reinterpret_cast<uint4*>(out), H / 8, vocab);
}

__global__ void gather_rows_kernel(const uint4* __restrict__ x, const int32_t* __restrict__ rows, uint4* __restrict__ out, int H8) {
    griddep_launch(); griddep_wait();
    const uint4* src = x + (size_t)rows[blockIdx.x] * H8;
    uint4* dst = out + (size_t)blockIdx.x * H8;
    for (int i = threadIdx.x; i < H8; i += blockDim.x) dst[i] = src[i];
}
cudaError_t launch_gather_rows(const void* x, const int32_t* rows, void* out, int n, int H, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    return launch_k(gather_rows_kernel, dim3(n), dim3(128), 0, s, reinterpret_cast<const uint4*>(x), rows, reinterpret_cast<uint4*>(out), H / 8);
}

// fp8 row quantiser: per row, s = w8_row_scale(max |x|) and q = e4m3(x * (1/s)) — exact division by a power of two, then RNE, saturating.
// One CTA per row; the second pass re-reads the row from L1 / L2.
__global__ void __launch_bounds__(256) quant_rows_e4m3_kernel(const uint4* __restrict__ x, uint2* __restrict__ q, float* __restrict__ scale, int C8) {
    griddep_launch(); griddep_wait();
    const uint4* xr = x + (size_t)blockIdx.x * C8;
    float amax = 0.f;
    for (int i = threadIdx.x; i < C8; i += blockDim.x) {
        float f[8];
        unpack_bf16x8(xr[i], f);
#pragma unroll
        for (int k = 0; k < 8; ++k) amax = fmaxf(amax, fabsf(f[k]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    __shared__ float red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < 8; ++w) amax = fmaxf(amax, red[w]);
    const float s = w8_row_scale(amax), inv = 1.0f / s;
    if (threadIdx.x == 0) scale[blockIdx.x] = s;
    uint2* qr = q + (size_t)blockIdx.x * C8;
    for (int i = threadIdx.x; i < C8; i += blockDim.x) {
        float f[8];
        unpack_bf16x8(xr[i], f);
        qr[i] = pack_e4m3x8(f, inv);
    }
}
cudaError_t launch_quant_rows_e4m3(const void* x, uint8_t* q, float* scale, int R, int C, cudaStream_t s) {
    if (R <= 0) return cudaSuccess;
    if (C <= 0 || C % 16 != 0) return cudaErrorInvalidValue;
    return launch_k(quant_rows_e4m3_kernel, dim3(R), dim3(256), 0, s, reinterpret_cast<const uint4*>(x), reinterpret_cast<uint2*>(q), scale, C / 8);
}

// y = x * rsqrt(mean(x^2) + eps) * g ; fp32 statistics, bf16 in/out.  Row cached in registers (H <= 8192).
template <int VPT>   // uint4 vectors per thread, 256 threads
__global__ void __launch_bounds__(256) rmsnorm_kernel(const uint4* __restrict__ x, const uint4* __restrict__ g, uint4* __restrict__ y,
                                                      int H8, float inv_h, float eps) {
    griddep_launch(); griddep_wait();
    const int t = blockIdx.x;
    const uint4* xr = x + (size_t)t * H8;
    uint4 v[VPT];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
        int i = threadIdx.x + k * 256;
        if (i < H8) {
            v[k] = xr[i];
            ss = sumsq_bf16x8(v[k], ss);
        }
    }
    ss = warp_sum(ss);
    __shared__ float red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += red[w];
    const float r = 1.0f / sqrtf(tot * inv_h + eps);
    uint4* yr = y + (size_t)t * H8;
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
        int i = threadIdx.x + k * 256;
        if (i < H8) yr[i] = rms_scale_bf16x8(v[k], r, g[i]);
    }
}
cudaError_t launch_rmsnorm(const void* x, const void* gain, void* y, int T, int H, float eps, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    if (H % 8 != 0 || H > 8192) return cudaErrorInvalidValue;
    const int H8 = H / 8;
    auto X = reinterpret_cast<const uint4*>(x); auto G = reinterpret_cast<const uint4*>(gain); auto Y = reinterpret_cast<uint4*>(y);
    if (H8 <= 256) return launch_k(rmsnorm_kernel<1>, dim3(T), dim3(256), 0, s, X, G, Y, H8, 1.0f / H, eps);
    if (H8 <= 512) return launch_k(rmsnorm_kernel<2>, dim3(T), dim3(256), 0, s, X, G, Y, H8, 1.0f / H, eps);
    return launch_k(rmsnorm_kernel<4>, dim3(T), dim3(256), 0, s, X, G, Y, H8, 1.0f / H, eps);
}

// One CTA per token.  Thread i handles the rotate-half pair group (8 consecutive i in [0,D/2) and the
// matching 8 in [D/2,D)) of one head: two 16-byte loads, two 16-byte stores.  a.bias is unused: qkv already holds the biased projection.
__global__ void rope_kv_write_kernel(const uint16_t* __restrict__ qkv, const SkRopeArgs a) {
    griddep_launch(); griddep_wait();
    const int t = blockIdx.x;
    const int D = a.D, half = D >> 1, vec_per_head = half >> 3;        // 8 pairs per thread
    const uint16_t* row = qkv + (size_t)t * (a.nh + 2 * a.nkv) * D;
    const int pos = a.positions[t];
    const int slot = a.slots[t];
    const int page = slot / a.page_size, off = slot - page * a.page_size;
    const float* cr = a.rope_cos + (size_t)pos * half;
    const float* sr = a.rope_sin + (size_t)pos * half;
    const int n_rot = (a.nh + a.nkv) * vec_per_head;
    for (int w = threadIdx.x; w < n_rot; w += blockDim.x) {
        const int head = w / vec_per_head, i0 = (w - head * vec_per_head) * 8;
        const uint16_t* src = row + (size_t)head * D;
        float av[8], bv[8];
        unpack_bf16x8(*reinterpret_cast<const uint4*>(src + i0), av);
        unpack_bf16x8(*reinterpret_cast<const uint4*>(src + i0 + half), bv);
        rope_store8(a, t, head, page, off, i0, av, bv, cr + i0, sr + i0);
    }
    // V: straight copy into the V plane
    const int n_v = a.nkv * (D >> 3);
    for (int w = threadIdx.x; w < n_v; w += blockDim.x) {
        const int head = w / (D >> 3), i0 = (w - head * (D >> 3)) * 8;
        kv_store8(a, t, a.nh + a.nkv + head, page, off, i0, *reinterpret_cast<const uint4*>(row + (size_t)(a.nh + a.nkv + head) * D + i0));
    }
}
cudaError_t launch_rope_kv_write(const void* qkv, const int32_t* positions, const int32_t* slots, const float* rope_cos,
                                 const float* rope_sin, void* q_out, const KvLayout& kv, int layer, int T, int nh, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    if (kv.head_dim % 16 != 0) return cudaErrorInvalidValue;
    return launch_k(rope_kv_write_kernel, dim3(T), dim3(256), 0, s, reinterpret_cast<const uint16_t*>(qkv),
                    make_sk_rope_args(nullptr, positions, slots, rope_cos, rope_sin, q_out, kv, layer, nh));
}


// =============================================================================================
// stream-K consumers (stand-alone kernels; the bodies live in sk_consumers.cuh)
// =============================================================================================
template <int VPT>
__global__ void __launch_bounds__(SK_RESID_THREADS) sk_resid_rmsnorm_kernel(const StreamK sk, uint4* __restrict__ x, const uint4* __restrict__ g,
                                                                            uint4* __restrict__ y, int H8, float inv_h, float eps) {
    griddep_launch(); griddep_wait();
    __shared__ float red[SK_RESID_THREADS / 32];
    sk_resid_rmsnorm_row<VPT>(sk, blockIdx.x, threadIdx.x, red, 0, x, g, y, H8, inv_h, eps);
}
cudaError_t launch_sk_resid_rmsnorm(const StreamK& sk, void* x, const void* gain, void* xn, int T, int H, float eps, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    if (H % 8 != 0 || H > 8192 || T > sk.rows) return cudaErrorInvalidValue;
    const int H8 = H / 8;
    auto X = reinterpret_cast<uint4*>(x); auto G = reinterpret_cast<const uint4*>(gain); auto Y = reinterpret_cast<uint4*>(xn);
    if (H8 <= SK_RESID_THREADS) return launch_k(sk_resid_rmsnorm_kernel<1>, dim3(T), dim3(SK_RESID_THREADS), 0, s, sk, X, G, Y, H8, 1.0f / H, eps);
    return launch_k(sk_resid_rmsnorm_kernel<2>, dim3(T), dim3(SK_RESID_THREADS), 0, s, sk, X, G, Y, H8, 1.0f / H, eps);
}

template <int VPT>
__global__ void __launch_bounds__(SK_RESID_THREADS) rmsnorm_wide_kernel(uint4* __restrict__ x, const uint4* __restrict__ g, uint4* __restrict__ y, int H8, float inv_h, float eps) {
    griddep_launch(); griddep_wait();
    __shared__ float red[SK_RESID_THREADS / 32];
    sk_resid_rmsnorm_row<VPT, false>(StreamK{}, blockIdx.x, threadIdx.x, red, 0, x, g, y, H8, inv_h, eps);
}
cudaError_t launch_rmsnorm_wide(const void* x, const void* gain, void* xn, int T, int H, float eps, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    if (H % 8 != 0 || H > 8192) return cudaErrorInvalidValue;
    const int H8 = H / 8;
    auto X = reinterpret_cast<uint4*>(const_cast<void*>(x)); auto G = reinterpret_cast<const uint4*>(gain); auto Y = reinterpret_cast<uint4*>(xn);
    if (H8 <= SK_RESID_THREADS) return launch_k(rmsnorm_wide_kernel<1>, dim3(T), dim3(SK_RESID_THREADS), 0, s, X, G, Y, H8, 1.0f / H, eps);
    return launch_k(rmsnorm_wide_kernel<2>, dim3(T), dim3(SK_RESID_THREADS), 0, s, X, G, Y, H8, 1.0f / H, eps);
}

__global__ void sk_swiglu_kernel(const StreamK sk, uint4* __restrict__ act, int F8) {
    griddep_launch(); griddep_wait();
    const int t = blockIdx.y;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < F8; i += gridDim.x * blockDim.x) sk_swiglu_item(sk, t, i, act, F8);
}
cudaError_t launch_sk_swiglu(const StreamK& sk, void* act, int T, int F, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    if (F % 16 != 0 || T > sk.rows) return cudaErrorInvalidValue;
    return launch_k(sk_swiglu_kernel, dim3((F / 8 + 255) / 256, T), dim3(256), 0, s, sk, reinterpret_cast<uint4*>(act), F / 8);
}

__global__ void sk_rope_kv_write_kernel(const StreamK sk, const SkRopeArgs a) {
    griddep_launch(); griddep_wait();
    const int t = blockIdx.y, items = sk_rope_items_per_row(a);
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < items; w += gridDim.x * blockDim.x) sk_rope_item(sk, a, t, w);
}
SkRopeArgs make_sk_rope_args(const void* bias, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin,
                             void* q_out, const KvLayout& kv, int layer, int nh) {
    SkRopeArgs a{};
    a.bias = reinterpret_cast<const uint16_t*>(bias); a.positions = positions; a.slots = slots; a.rope_cos = rope_cos; a.rope_sin = rope_sin;
    a.q_out = reinterpret_cast<uint16_t*>(q_out); a.kv_base = reinterpret_cast<uint16_t*>(kv.base);
    a.k_plane_row0 = (int64_t)layer * kv.layer_stride_rows; a.v_plane_row0 = a.k_plane_row0 + kv.kv_stride_rows;
    a.page_size = kv.page_size; a.nh = nh; a.nkv = kv.n_kv; a.D = kv.head_dim;
    a.kv_fp8 = kv.fp8;
    if (kv.fp8) { a.k_inv_scale = 1.0f / kv.k_scale[layer]; a.v_inv_scale = 1.0f / kv.v_scale[layer]; }
    return a;
}
cudaError_t launch_sk_rope_kv_write(const StreamK& sk, const void* bias, const int32_t* positions, const int32_t* slots,
                                    const float* rope_cos, const float* rope_sin, void* q_out, const KvLayout& kv, int layer, int T,
                                    int nh, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    if (kv.head_dim % 16 != 0 || T > sk.rows) return cudaErrorInvalidValue;
    const SkRopeArgs a = make_sk_rope_args(bias, positions, slots, rope_cos, rope_sin, q_out, kv, layer, nh);
    const int items = (nh + kv.n_kv) * (kv.head_dim / 16) + kv.n_kv * (kv.head_dim / 8);
    return launch_k(sk_rope_kv_write_kernel, dim3((items + 127) / 128, T), dim3(128), 0, s, sk, a);
}

}  // namespace oa
