// common.cuh — device-side building blocks for sm_90a: bf16 helpers, mbarrier, TMA, wgmma,
// ldmatrix/mma.sync wrappers.  Everything here is inline PTX; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define OA_DEVINL __device__ __forceinline__

namespace oa {

// ---------------------------------------------------------------------------------------------
// bf16 <-> fp32 with the exact bit logic of oracle/llama_ref.c (round-to-nearest-even)
// ---------------------------------------------------------------------------------------------
__host__ OA_DEVINL uint16_t f32_to_bf16_bits(float f) {
    uint32_t u;
#ifdef __CUDA_ARCH__
    u = __float_as_uint(f);
#else
    memcpy(&u, &f, 4);
#endif
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
    uint32_t r = 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)((u + r) >> 16);
}
OA_DEVINL float bf16_bits_to_f32(uint16_t h) { return __uint_as_float(((uint32_t)h) << 16); }
OA_DEVINL float bf16lo(uint32_t packed) { return __uint_as_float(packed << 16); }
OA_DEVINL float bf16hi(uint32_t packed) { return __uint_as_float(packed & 0xffff0000u); }
// pack two fp32 -> bf16x2 (lo = a, hi = b), RNE (cvt.rn.bf16x2.f32 takes hi operand first)
OA_DEVINL uint32_t pack_bf16x2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}

// ---------------------------------------------------------------------------------------------
// Epilogue arithmetic on 8 bf16 lanes (one 16-byte vector).  Every GEMM epilogue and every consumer kernel finishes its values
// with these, so the fused and the stand-alone paths perform the same fp32 operations in the same order (bit-identical results).
// ---------------------------------------------------------------------------------------------
OA_DEVINL void unpack_bf16x8(uint4 u, float* f) {
    f[0] = bf16lo(u.x); f[1] = bf16hi(u.x); f[2] = bf16lo(u.y); f[3] = bf16hi(u.y);
    f[4] = bf16lo(u.z); f[5] = bf16hi(u.z); f[6] = bf16lo(u.w); f[7] = bf16hi(u.w);
}
OA_DEVINL uint4 pack_bf16x8(const float* f) {
    uint4 o;
    o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]); o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
    return o;
}
// f[i] += bf16 lane i of u (bias or residual)
OA_DEVINL void add_bf16x8(float* f, uint4 u) {
    f[0] += bf16lo(u.x); f[1] += bf16hi(u.x); f[2] += bf16lo(u.y); f[3] += bf16hi(u.y);
    f[4] += bf16lo(u.z); f[5] += bf16hi(u.z); f[6] += bf16lo(u.w); f[7] += bf16hi(u.w);
}
// f[i] = bf16(f[i]) as fp32: a projection output that is a bf16 tensor
OA_DEVINL void round_bf16x8(float* f) {
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = bf16_bits_to_f32(f32_to_bf16_bits(f[k]));
}
// silu(g) * u, packed
OA_DEVINL uint4 swiglu_bf16x8(const float* g, const float* u) {
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = __fdividef(g[k], 1.0f + __expf(-g[k])) * u[k];
    return pack_bf16x8(f);
}
// RoPE (rotate-half pairing) of 8 (lo, hi) pairs with cos / sin rows cs, sn (16-byte aligned): lo·c − hi·s and hi·c + lo·s, packed
OA_DEVINL void rope_bf16x8(const float* lo, const float* hi, const float* cs, const float* sn, uint4& out_lo, uint4& out_hi) {
    const float4 c0 = *reinterpret_cast<const float4*>(cs), c1 = *reinterpret_cast<const float4*>(cs + 4);
    const float4 s0 = *reinterpret_cast<const float4*>(sn), s1 = *reinterpret_cast<const float4*>(sn + 4);
    const float cv[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    float ra[8], rb[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { ra[k] = lo[k] * cv[k] - hi[k] * sv[k]; rb[k] = hi[k] * cv[k] + lo[k] * sv[k]; }
    out_lo = pack_bf16x8(ra);
    out_hi = pack_bf16x8(rb);
}
// RMSNorm: ss + the squares of the 8 lanes of v, in lane order; and pack(v * r * g)
OA_DEVINL float sumsq_bf16x8(uint4 v, float ss) {
    float f[8];
    unpack_bf16x8(v, f);
#pragma unroll
    for (int k = 0; k < 8; ++k) ss += f[k] * f[k];
    return ss;
}
OA_DEVINL uint4 rms_scale_bf16x8(uint4 v, float r, uint4 g) {
    float a[8], b[8];
    unpack_bf16x8(v, a);
    unpack_bf16x8(g, b);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = a[k] * r * b[k];
    return pack_bf16x8(a);
}
// first element of row (page, kv head, offset in page) of a K or V plane starting at row plane_row0 of the paged cache (rows of D)
OA_DEVINL uint16_t* kv_row(uint16_t* kv_base, int64_t plane_row0, int page, int nkv, int head, int page_size, int off, int D) {
    return kv_base + (size_t)(plane_row0 + ((int64_t)page * nkv + head) * page_size + off) * D;
}
// fp8 KV cache (e4m3, OCP "fn" variant).  Four fp32 -> four bytes (byte i = lane i), round to nearest even, saturating to +-448: the
// NaN codes 0x7f / 0xff are never written.  cvt.*x2 takes the high operand first.
OA_DEVINL uint32_t pack_e4m3x4(float a, float b, float c, float d) {
    uint16_t lo, hi;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
    return (uint32_t)lo | ((uint32_t)hi << 16);
}
// 8 fp32 times `mul` -> 8 e4m3 bytes
OA_DEVINL uint2 pack_e4m3x8(const float* f, float mul) {
    return make_uint2(pack_e4m3x4(f[0] * mul, f[1] * mul, f[2] * mul, f[3] * mul), pack_e4m3x4(f[4] * mul, f[5] * mul, f[6] * mul, f[7] * mul));
}
// two e4m3 bytes (lo = byte 0) -> bf16x2, exact: every e4m3 value is an f16 normal or zero, and every f16 value of that set a bf16 value
OA_DEVINL uint32_t e4m3x2_to_bf16x2(uint16_t v) {
    uint32_t h;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(v));
    float lo, hi;
    asm("{\n\t.reg .f16 l, u;\n\tmov.b32 {l, u}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, u;\n\t}" : "=f"(lo), "=f"(hi) : "r"(h));
    return pack_bf16x2(lo, hi);
}

OA_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch: every kernel of the forward chain is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization.  griddep_launch() lets the next kernel's CTAs become resident and
// run their prologue (and, in the GEMMs, start streaming WEIGHTS, which no predecessor writes); griddep_wait() blocks
// until every predecessor grid has completed and its memory is visible — nothing produced by a predecessor may be
// touched, and nothing a predecessor reads may be written, before it.
// ---------------------------------------------------------------------------------------------
OA_DEVINL void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
OA_DEVINL void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
OA_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
OA_DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
OA_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
OA_DEVINL void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }    // generic-proxy global writes -> later TMA (async proxy) reads
// grid-wide counter barrier for persistent kernels whose CTAs are all co-resident (grid <= SM count, one CTA per SM)
OA_DEVINL unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
OA_DEVINL void grid_counter_wait(const unsigned long long* ctr, unsigned long long target) {
    uint32_t spins = 0;
    while (ld_acquire_gpu_u64(ctr) < target) {
        __nanosleep(20);
        if (++spins > (1u << 26)) { __trap(); }      // a protocol bug traps instead of hanging the GPU
    }
}
OA_DEVINL void grid_counter_wait32(const unsigned int* ctr, unsigned int target) {
    uint32_t spins = 0;
    unsigned int v;
    do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
        if (v >= target) break;
        __nanosleep(20);
        if (++spins > (1u << 26)) { __trap(); }
    } while (true);
}
OA_DEVINL void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
OA_DEVINL void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
OA_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (kernel error reported to the host) instead of hanging the GPU.
#ifndef OA_MBAR_SPIN_LIMIT
#define OA_MBAR_SPIN_LIMIT (1u << 26)
#endif
OA_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > OA_MBAR_SPIN_LIMIT) { __trap(); }
    }
}

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — 2D tiled loads completing on an mbarrier
// ---------------------------------------------------------------------------------------------
OA_DEVINL void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// L2 cache-policy constants (same encodings CUTLASS uses for TMA::CacheHintSm90)
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
OA_DEVINL void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0, int32_t c1, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
        : "memory");
}

// L2 prefetch of one tensor-map box (no smem destination, no barrier)
OA_DEVINL void tma_prefetch_l2_2d(const void* tmap, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];"
                 ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1) : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (Hopper warpgroup MMA): D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, bf16 operands K-major in shared memory, fp32
// accumulators in the registers of the issuing warpgroup (4 aligned warps, 128 threads, all of which execute every call).
// Fragment of m64nN: register r of thread (warp w of the warpgroup, lane l) holds
//   row = 16w + l/4 + 8*((r >> 1) & 1),  col = 8*(r >> 2) + 2*(l & 3) + (r & 1).
// ---------------------------------------------------------------------------------------------
OA_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
OA_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
OA_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptor of a K-major operand tile stored as rows of 128 B with the 128-byte swizzle (what a TMA box
// {64 bf16, rows} with CU_TENSOR_MAP_SWIZZLE_128B produces): start address >>4 in [0,14); LBO (unused for swizzled K-major) = 1
// in [16,30); SBO = 1024 B (8 rows x 128 B) >>4 in [32,46); layout SWIZZLE_128B = 1 in [62,64).  Stepping 16 bf16 (32 B) along K
// inside the swizzle row is +2 in the address field.
OA_DEVINL uint64_t gmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

#define OA_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define OA_F16(i) OA_F4(i), OA_F4(i + 4), OA_F4(i + 8), OA_F4(i + 12)
OA_DEVINL void wgmma_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : OA_F16(0)
        : "l"(da), "l"(db), "r"(acc) : "memory");
}
OA_DEVINL void wgmma_m64n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : OA_F16(0), OA_F16(16)
        : "l"(da), "l"(db), "r"(acc) : "memory");
}
OA_DEVINL void wgmma_m64n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : OA_F16(0), OA_F16(16), OA_F16(32), OA_F16(48)
        : "l"(da), "l"(db), "r"(acc) : "memory");
}
// MN-major operand (e.g. V[kv, d] with d contiguous used as B[N = d, K = kv]), 128-byte swizzle: atoms of 64 N-elements x 8 K-rows
// (1024 B); LBO = byte stride between 64-element N blocks, SBO = byte stride between 8-row K groups.
OA_DEVINL uint64_t gmma_desc_sw128_mn(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// A from registers (4 x bf16x2 per thread, the mma.sync m16n8k16 A-fragment layout for the warp's 16 rows); *_tb: B MN-major
OA_DEVINL void wgmma_rs_m64n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : OA_F16(0), OA_F16(16)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc) : "memory");
}
OA_DEVINL void wgmma_rs_m64n64_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
        : OA_F16(0), OA_F16(16)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc) : "memory");
}
OA_DEVINL void wgmma_rs_m64n128_tb(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1, 1;\n\t}"
        : OA_F16(0), OA_F16(16), OA_F16(32), OA_F16(48)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc) : "memory");
}
OA_DEVINL void wgmma_rs_m64n128(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : OA_F16(0), OA_F16(16), OA_F16(32), OA_F16(48)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc) : "memory");
}
template <int N>
OA_DEVINL void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc) {
    if constexpr (N == 32) wgmma_m64n32(d, da, db, acc);
    else if constexpr (N == 64) wgmma_m64n64(d, da, db, acc);
    else { static_assert(N == 128, "wgmma N in {32, 64, 128}"); wgmma_m64n128(d, da, db, acc); }
}
// D[64 x N] (+)= A[64 x 32] . B[N x 32]^T with e4m3 operands (both K-major, same descriptors: 32 bytes of K per instruction), fp32 out.
// The tensor core keeps only about 14 mantissa bits of the running sum across the k32 steps: callers sum a few steps here and promote.
OA_DEVINL void wgmma_e4m3_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, %16, %17, p, 1, 1;\n\t}"
        : OA_F16(0)
        : "l"(da), "l"(db), "r"(acc) : "memory");
}
OA_DEVINL void wgmma_e4m3_m64n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1;\n\t}"
        : OA_F16(0), OA_F16(16)
        : "l"(da), "l"(db), "r"(acc) : "memory");
}
OA_DEVINL void wgmma_e4m3_m64n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1;\n\t}"
        : OA_F16(0), OA_F16(16), OA_F16(32), OA_F16(48)
        : "l"(da), "l"(db), "r"(acc) : "memory");
}
template <int N>
OA_DEVINL void wgmma_e4m3(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc) {
    if constexpr (N == 32) wgmma_e4m3_m64n32(d, da, db, acc);
    else if constexpr (N == 64) wgmma_e4m3_m64n64(d, da, db, acc);
    else { static_assert(N == 128, "wgmma N in {32, 64, 128}"); wgmma_e4m3_m64n128(d, da, db, acc); }
}
// Row scale of the fp8 (e4m3) projections and their inputs: the smallest power of two s with amax <= 448 * s (amax = 0: 1), as a normal
// fp32.  From the bits of amax = 1.f * 2^(e-127): 448 * 2^(e-135) = 1.75 * 2^(e-127), so s = 2^(e-135) when 1.f <= 1.75, else 2^(e-134).
__host__ OA_DEVINL float w8_row_scale(float amax) {
    uint32_t u;
#ifdef __CUDA_ARCH__
    u = __float_as_uint(amax);
#else
    memcpy(&u, &amax, 4);
#endif
    u &= 0x7fffffffu;
    if (u == 0) return 1.0f;
    const int e = (int)(u >> 23);
    int k = e == 0 ? -126 : e - 135 + ((u & 0x7fffffu) > 0x600000u ? 1 : 0);
    k = k < -126 ? -126 : k;
    const uint32_t sb = (uint32_t)(k + 127) << 23;
#ifdef __CUDA_ARCH__
    return __uint_as_float(sb);
#else
    float s; memcpy(&s, &sb, 4); return s;
#endif
}

// fp32 accumulator tile [rows][N] in shared memory, 16-byte chunks XOR-swizzled by (row & 7): a warp storing its wgmma fragment
// and a warp reading 32 consecutive columns of 32 rows (one row per lane) are both free of bank conflicts.  N >= 32.
OA_DEVINL int acc_idx(int N, int row, int col) { return row * N + ((((col >> 2) ^ row) & 7) | ((col >> 2) & ~7)) * 4 + (col & 3); }
// warpgroup fragment of rows [row0, row0 + 64) -> the shared tile
template <int N>
OA_DEVINL void acc_store_frag(float* acc, int row0, const float (&d)[N / 2]) {
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = row0 + 16 * w + (lane >> 2) + 8 * h, col = 8 * j + 2 * (lane & 3);
            *reinterpret_cast<float2*>(acc + acc_idx(N, row, col)) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
        }
    }
}
OA_DEVINL float4 acc_ld4(const float* acc, int N, int row, int col) { return *reinterpret_cast<const float4*>(acc + acc_idx(N, row, col)); }
// one row x 32 columns [col0, col0 + 32) (col0 % 32 == 0) as raw fp32 bits
OA_DEVINL void acc_ld32(const float* acc, int N, int row, int col0, uint32_t (&v)[32]) {
#pragma unroll
    for (int c = 0; c < 32; c += 4) {
        const float4 x = acc_ld4(acc, N, row, col0 + c);
        v[c] = __float_as_uint(x.x); v[c + 1] = __float_as_uint(x.y); v[c + 2] = __float_as_uint(x.z); v[c + 3] = __float_as_uint(x.w);
    }
}

// ---------------------------------------------------------------------------------------------
// legacy warp-level tensor path (used by the HBM-bound attention kernels: 16-row tiles)
// ---------------------------------------------------------------------------------------------
OA_DEVINL void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
OA_DEVINL void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
// D(16x8,f32) += A(16x16,bf16,row) * B(16x8,bf16,col)
OA_DEVINL void mma_bf16_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// 2^x on the SFU, flush-to-zero, no range fix-up code around it (inputs here are <= ~8; -inf -> 0)
OA_DEVINL float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

OA_DEVINL float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Arg-max of row `row` of per-tile (value, column) partials [rows, n_tiles] over one block of <= 256 threads: the larger value wins, the
// lower column on ties.  The result is in thread 0's (bv, bi); bi = 0x7fffffff when the row has no candidate.
OA_DEVINL void block_argmax_row(const float* __restrict__ val, const int* __restrict__ idx, int row, int n_tiles, float& bv, int& bi) {
    bv = -INFINITY; bi = 0x7fffffff;
    for (int t = threadIdx.x; t < n_tiles; t += blockDim.x) {
        const float v = val[(size_t)row * n_tiles + t]; const int i = idx[(size_t)row * n_tiles + t];
        if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    __shared__ float sv[8]; __shared__ int si[8];
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
            if (sv[w] > bv || (sv[w] == bv && si[w] < bi)) { bv = sv[w]; bi = si[w]; }
    }
}

// 16-byte global accesses
OA_DEVINL uint4 ld_nc_16(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

}  // namespace oa
