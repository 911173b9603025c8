// tma.cpp — CUtensorMap construction.  cuTensorMapEncodeTiled is resolved through the CUDA runtime
// (cudaGetDriverEntryPoint) so the library has no link-time dependency on libcuda.so and loads on a
// GPU-less build box.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "kernels.hpp"

namespace oa {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn resolve_encode() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems,
                      uint32_t box_rows, uint32_t box_cols) {
    EncodeTiledFn enc = resolve_encode();
    if (!enc) return -1;
    if (box_cols * 2 > 128 || box_rows > 256 || (pitch_elems * 2) % 16 != 0 || (reinterpret_cast<uintptr_t>(base) & 15)) return -2;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {pitch_elems * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

int make_tmap_u8_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols) {
    EncodeTiledFn enc = resolve_encode();
    if (!enc) return -1;
    if (box_cols > 128 || box_rows > 256 || cols % 16 != 0 || (reinterpret_cast<uintptr_t>(base) & 15)) return -2;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {cols};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

static std::atomic<uint64_t> g_launches{0};
uint64_t launches_total() { return g_launches.load(); }
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
bool pdl_enabled() {
    static const bool on = [] { const char* e = std::getenv("OA_PDL"); return !(e && e[0] == '0'); }();
    return on;
}

}  // namespace oa
