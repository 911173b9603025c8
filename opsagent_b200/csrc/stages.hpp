// stages.hpp — the launch sequences of DeviceModel::forward, one function per stage, called by the forward and by the kernel test entry
// points (capi_kernels.cpp) alike, so the kernel tests run what serves traffic.  Asynchronous on `s`; a failed launch throws CudaError.
#pragma once
#include <functional>
#include <stdexcept>
#include <string>

#include "kernels.hpp"
#include "tp_comm.hpp"

namespace oa {

struct CudaError : std::runtime_error {      // cuda_check's "<what>: <CUDA error string>", with the error
    cudaError_t code;
    CudaError(cudaError_t e, const std::string& msg) : std::runtime_error(msg), code(e) {}
};
void cuda_check(cudaError_t e, const char* what);
// OA_PROFILE_ALL: called with the kernel class (DeviceModel::kt_name) after a stage's launches; empty: no marks
using Mark = std::function<void(int)>;

// A decode projection A.B^T [M, N].  path 0 = stream-K GEMM (BLOCK_N sk.bn) + consumer, 1 = consumer fused into the GEMM (BLOCK_N 128,
// tile_flags), >= 2 = cluster split-K of that size (bf16, BLOCK_N 128).  Only the GEMM reads sk.l2_prefetch_units.
struct SkGemm { int path; const CUtensorMap *tmA, *tmB; int M, N, K; StreamK sk; W8Scales w8; unsigned int* tile_flags; };
// Row-parallel projections (o, down): the kernel class of the GEMM and the cuda_check labels
struct RowParallelOp { int mark; const char *clusterk, *fused, *gemm, *norm, *resid, *nvls_part, *nvls_ar, *bf16_part, *f32_part, *ar; };
extern const RowParallelOp kOProj, kDownProj;
// single GPU: x [M, N] += A.B^T, then xn = rmsnorm(x) * gain
void finish_row_parallel(const SkGemm& g, void* x, const void* gain, void* xn, float eps, const RowParallelOp& op, cudaStream_t s, const Mark& mark = {});
// tensor parallel (path 0), split at the cross-rank wait.  Producer: the GEMM, then its fp32 / bf16 sum into `partial` and the signal
void tp_row_parallel_partial(const SkGemm& g, bool bf16, void* partial, const TpComm::Signal& sg, const RowParallelOp& op, cudaStream_t s,
                             const Mark& mark = {});
// consumer: after the t ranks' signals, x += the rank-ordered sum of the partials (device table), then xn = rmsnorm(x) * gain
void tp_row_parallel_finish(void* const* peer_partials, int t, bool bf16, void* x, const void* gain, void* xn, int M, int N, float eps,
                            const TpComm::Signal& sg, const RowParallelOp& op, cudaStream_t s, const Mark& mark = {});
// qkv (+ bias) -> bf16 -> RoPE -> q_out and layer `layer` of the paged cache
void qkv_rope(const SkGemm& g, const void* bias, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin,
              void* q_out, const KvLayout& kv, int layer, int nh, cudaStream_t s, const Mark& mark = {});
// gate/up [M, N = 2F] -> act [M, F] = silu(gate) * up; paths 0 and 1
void gate_up_swiglu(const SkGemm& g, void* act, cudaStream_t s, const Mark& mark = {});

// One layer's attention: decode attention (when dec.n_ctas > 0), then prefill attention (when pre.n_tiles > 0), both at `layer` and scale_log2e
void step_attention(const CUtensorMap* tm_kv, const KvLayout& kv, DecodeAttnParams dec, PrefillAttnParams pre, int layer, cudaStream_t s,
                    const Mark& mark = {});

// LM head: the EPI_LOGITS GEMM [M, N] (per-tile row maxima, logits when non-null, mask rows as GemmParams), then ids [M] = the row arg-max,
// or for a vocab shard (pair_out) its (max, col_offset + arg-max) pair per row
void lm_head_argmax(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int bn, float* logits, int ldl, float* amax_val,
                    int* amax_idx, const uint32_t* mask_table, const int32_t* mask_slot, int mask_words, int col_offset, int32_t* ids,
                    void* pair_out, cudaStream_t s, const Mark& mark = {});

// tile-path projection: EPI_STORE out (+ bias), EPI_RESID out = resid + A.B^T (the forward: resid = out), EPI_SWIGLU out [M, N/2]
void proj_gemm(const CUtensorMap* tmA, const CUtensorMap* tmB, int M, int N, int K, int epilogue, int bn, void* out, const void* bias,
               const void* resid, W8Scales w8, const char* label, cudaStream_t s);

}  // namespace oa
