// weights.cu — deterministic seeded weight initialisation on the device.  The generator is the one in
// oracle/llama_ref.c (mix64 -> Irwin-Hall(4) of 16-bit uniforms -> one fp32 multiply-add -> bf16 RNE):
// integer arithmetic plus exactly-rounded fp32 ops, so both sides produce identical bf16 bits.
#include "common.cuh"
#include "kernels.hpp"

namespace oa {

OA_DEVINL uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
OA_DEVINL uint16_t gen_bf16(uint64_t key, uint64_t idx, float std, float mean) {
    uint64_t h = mix64(key + idx);
    int32_t s = (int32_t)(h & 0xffff) + (int32_t)((h >> 16) & 0xffff) + (int32_t)((h >> 32) & 0xffff) +
                (int32_t)((h >> 48) & 0xffff) - 131070;
    // separate multiply and add (no FMA contraction) to match the C oracle compiled without -ffp-contract
    float u = __fmul_rn((float)s, 1.0f / 37837.227f);
    return f32_to_bf16_bits(__fadd_rn(__fmul_rn(u, std), mean));
}

// (row_off, col_off, logical_cols) place this (possibly tensor-parallel) shard inside the logical tensor, so every rank
// generates exactly the slice of the single-GPU tensor it owns.
__global__ void init_weight_kernel(uint16_t* __restrict__ dst, uint64_t key_a, uint64_t key_b, int interleave, int64_t rows,
                                   int64_t cols, float std, float mean, int64_t row_off, int64_t col_off, int64_t logical_cols) {
    const int64_t n = rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = i / cols, c = i - r * cols;
        uint64_t key = key_a; int64_t lr = r;
        if (interleave) {              // fused gate/up: 16 gate rows then 16 up rows per 32-row block
            int64_t blk = r >> 5, w = r & 31;
            lr = blk * 16 + (w & 15);
            key = (w < 16) ? key_a : key_b;
        }
        dst[i] = gen_bf16(key, (uint64_t)((lr + row_off) * logical_cols + col_off + c), std, mean);
    }
}

static uint64_t host_mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

cudaError_t launch_init_weight(void* dst, uint64_t seed, uint64_t tensor_id, int64_t tensor_id_b, int64_t rows, int64_t cols,
                               float std, float mean, cudaStream_t s, int64_t row_off, int64_t col_off, int64_t logical_cols) {
    if (logical_cols <= 0) logical_cols = cols;
    uint64_t key_a = host_mix64(seed ^ (tensor_id * 0xD6E8FEB86659FD93ull));
    uint64_t key_b = tensor_id_b >= 0 ? host_mix64(seed ^ ((uint64_t)tensor_id_b * 0xD6E8FEB86659FD93ull)) : 0;
    int64_t n = rows * cols;
    int blocks = (int)((n + 255) / 256 < 132 * 16 ? (n + 255) / 256 : 132 * 16);
    init_weight_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<uint16_t*>(dst), key_a, key_b, tensor_id_b >= 0 ? 1 : 0, rows, cols,
                                              std, mean, row_off, col_off, logical_cols);
    count_launch();
    return cudaGetLastError();
}

}  // namespace oa
