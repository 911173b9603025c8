// tp_comm.hpp — tensor-parallel plumbing for models that do not fit one GPU (BASELINE configs[3,4]).
//
// One process per GPU on one NVSwitch node.  No NCCL: ranks exchange CUDA-IPC handles of *symmetric* buffers through a
// POSIX shared-memory segment, map each other's buffers, and the row-parallel projections are all-reduced by the
// engine's own kernels reading peer memory over NVLink (tp_comm.cu):
//     partial -> own symmetric buffer;  xgpu_barrier (release/acquire flags in peer memory);
//     every rank adds the t partials in RANK ORDER (bit-identical result on all ranks) fused with residual add + RMSNorm.
// Rank 0 (leader) owns the scheduler; each step it publishes the packed step metadata in the shm segment and the
// followers replay the same forward — they hold no request state.
#pragma once
#include <atomic>
#include <cstdint>
#include <string>
#include <vector>

#include "kernels.hpp"

namespace oa {

struct StepInput;

constexpr int TP_MAX = 8;
constexpr size_t TP_MSG_WORDS = 2u << 20;     // 8 MB step-message area

struct TpShm {                                 // lives in POSIX shared memory
    std::atomic<uint32_t> magic;               // set LAST by the leader; cleared first thing when a new leader finds a stale segment
    std::atomic<uint64_t> nonce;               // per-launch id (config "tp_nonce"): followers refuse a segment of another launch
    std::atomic<int64_t> leader_pid;
    std::atomic<int64_t> rank_pid[TP_MAX];
    std::atomic<uint32_t> nvls_leader_ready;   // multicast setup (tp_nvls.cpp): 0 pending, 1 the leader's fd server is up, 2 the leader could not create the object
    std::atomic<uint32_t> nvls_stage[2];       // ranks that finished a setup stage
    std::atomic<uint32_t> nvls_fail;           // ranks that failed at any stage: > 0 -> every rank falls back to the peer-memory all-reduce     // every rank's pid (set when it attaches): the leader notices a follower that died instead of waiting out a timeout           // followers refuse a segment whose leader is gone and notice a leader that dies later
    std::atomic<uint32_t> handles_ready;       // ranks that published their IPC handles
    std::atomic<uint32_t> peers_opened;        // ranks that mapped every peer
    cudaIpcMemHandle_t h_sym[TP_MAX][3];       // [rank][buffer]: 0/1 = double-buffered partials, 2 = the gather buffer of the two-shot all-reduce
    cudaIpcMemHandle_t h_flags[TP_MAX];
    cudaIpcMemHandle_t h_arg[TP_MAX];
    std::atomic<uint64_t> seq;                 // step message sequence (UINT64_MAX = shutdown)
    std::atomic<uint64_t> ack[TP_MAX];
    uint32_t msg_words;
    int32_t msg[TP_MSG_WORDS];
};

class TpComm {
public:
    // nvls_bytes > 0: also try to set up an NVLink-switch multicast buffer of that size (in-switch all-reduce); nvls() tells whether every rank succeeded
    TpComm(int t, int rank, const std::string& shm_name, size_t sym_bytes, int max_sample, uint64_t nonce = 0, size_t nvls_bytes = 0);
    ~TpComm();
    int size() const { return t_; }
    int rank() const { return rank_; }

    // ---- device side ----
    int next_buffer() { return (int)(ar_count_++ & 1); }                // double-buffered symmetric storage
    void* sym(int b) const { return sym_[b]; }                            // this rank's buffer b (0/1: partials, alternating; 2: gather buffer)
    static constexpr int GATHER = 2;
    // in-switch (NVLS) buffer: this rank's copy at a unicast address, the multicast address spanning every rank's copy
    bool nvls() const { return nvls_uc_ != nullptr; }
    void* nvls_local() const { return nvls_uc_; }
    void* nvls_multicast() const { return nvls_mc_; }
    size_t nvls_bytes() const { return nvls_bytes_; }
    void* const* d_peer_sym(int b) const { return d_peer_sym_[b]; }       // device array [t] of peer pointers for buffer b
    void* peer_sym_host(int b, int p) const { return peer_sym_[b][p]; }
    size_t sym_bytes() const { return sym_bytes_; }
    void* arg(int b) const { return reinterpret_cast<char*>(arg_) + (size_t)b * arg_half_bytes_; }
    void* const* d_peer_arg(int b) const { return d_peer_arg_[b]; }
    cudaError_t barrier(cudaStream_t s);                                  // every rank's prior writes visible to all
    // the same handshake split over two kernels: the producer's last CTA signals "my buffer is written" to every peer, the
    // consumer's CTAs wait for every peer's signal before their first peer load (no stand-alone barrier launch)
    struct Signal { uint32_t* const* peer_flags; const uint32_t* my_flags; unsigned int* done_counter; int rank, t; uint32_t epoch; };
    Signal next_signal() { ++epoch_; return Signal{(uint32_t* const*)d_peer_flags_, flags_, done_counter_, rank_, t_, epoch_}; }

    // ---- host side: leader publishes, followers receive ----
    void publish(const StepInput& in);
    bool receive(StepInput& in);                                          // false = shutdown; throws when the leader process has died
    bool leader_alive() const;
    void shutdown();

private:
    bool nvls_setup(size_t bytes_wanted, uint64_t nonce);      // tp_nvls.cpp
    void nvls_teardown();
    void* nvls_uc_ = nullptr; void* nvls_mc_ = nullptr; size_t nvls_bytes_ = 0; unsigned long long nvls_mem_ = 0, nvls_obj_ = 0;
    int t_, rank_; std::string shm_name_; TpShm* shm_ = nullptr; bool owner_ = false;
    void* sym_[3] = {nullptr, nullptr, nullptr}; void* peer_sym_[3][TP_MAX] = {};
    void** d_peer_sym_[3] = {nullptr, nullptr, nullptr};
    uint32_t* flags_ = nullptr; uint32_t* peer_flags_[TP_MAX] = {}; uint32_t** d_peer_flags_ = nullptr; unsigned int* done_counter_ = nullptr;
    void* arg_ = nullptr; void* peer_arg_[TP_MAX] = {}; void** d_peer_arg_[2] = {nullptr, nullptr}; size_t arg_half_bytes_ = 0;
    uint64_t ar_count_ = 0; uint32_t epoch_ = 0; uint64_t seq_local_ = 0; uint64_t idle_polls_ = 0; size_t sym_bytes_ = 0;
};

// x[T,H] (bf16, in place) += sum over ranks (rank order) of fp32 partial rows; xn = rmsnorm(x) * gain   (decode path)
// `wait` != null: every CTA first waits for all peers' signals of that epoch (TpComm::next_signal) instead of a preceding barrier launch
cudaError_t launch_ar_resid_rmsnorm(void* const* d_peer, int t, void* x, const void* gain, void* xn, int T, int H, float eps, cudaStream_t s,
                                    const TpComm::Signal* wait = nullptr);
// In-switch variant (NVLS): every rank's fp32 partial sits in its copy of the multicast buffer at `part_off`.  Token row c is owned by rank c % t:
// the owner asks the switch for the row's SUM over all ranks (multimem.ld_reduce), broadcasts it into every copy at `red_off` (multimem.st) and then
// broadcasts the row's flag (uint32 epochs at `flag_off`, multimem.st.release); every rank finishes residual + RMSNorm of row c from its LOCAL copy
// once its local flag shows the epoch.  2/t of a partial crosses a rank's links instead of t-1 partials; `wait` = peers' partials are written.
cudaError_t launch_ar_nvls_resid_rmsnorm(const void* mc_base, const void* local_base, size_t part_off, size_t red_off, size_t flag_off, int t, int rank, void* x,
                                         const void* gain, void* xn, int T, int H, float eps, cudaStream_t s, const TpComm::Signal& wait);
// the same with bf16 partial rows (half the NVLink bytes; engine option tp_ar_bf16)
cudaError_t launch_ar_resid_rmsnorm_bf16in(void* const* d_peer, int t, void* x, const void* gain, void* xn, int T, int H, float eps, cudaStream_t s,
                                           const TpComm::Signal* wait = nullptr);
cudaError_t launch_sk_reduce_bf16(const StreamK& sk, void* out, int T, int N, cudaStream_t s, const TpComm::Signal* signal = nullptr);
// x[T,H] += sum over ranks of bf16 partial rows                                                          (prefill path)
cudaError_t launch_ar_resid_bf16(void* const* d_peer, int t, void* x, int T, int H, cudaStream_t s);
// Two-shot variant for large T (prefill chunks): the one-shot kernel above makes every rank read all t full partials — t x T x H x 2 bytes, 1.07 GB
// per all-reduce for a Llama-3-70B TP=8 chunk of 8192 tokens, 160 times per chunk.  Here rank r reduces only slice r
// (reduce-scatter: reads (t-1)/t of ONE partial's bytes), adds the residual and publishes the finished bf16 slice in its gather buffer; after a
// barrier every rank copies the other t-1 slices (all-gather).  2 x (t-1)/t x T x H x 2 bytes per rank instead of (t-1) x T x H x 2; each element
// is computed once, by its slice owner, in rank order — all ranks still hold bit-identical activations.
cudaError_t launch_ar2_reduce_scatter(void* const* d_peer_partial, int t, int rank, void* x, void* gather_mine, int T, int H, cudaStream_t s);
cudaError_t launch_ar2_all_gather(void* const* d_peer_gather, int t, int rank, void* x, int T, int H, cudaStream_t s);
// stream-K partials -> fp32 rows [T,N] in `out` (this rank's symmetric buffer)
// `signal` != null: the last CTA to finish tells every peer that this rank's buffer is complete
cudaError_t launch_sk_reduce_f32(const StreamK& sk, float* out, int T, int N, cudaStream_t s, const TpComm::Signal* signal = nullptr);
// vocab-parallel greedy sampling: (val, global idx) per row into this rank's arg buffer, then combine over ranks
cudaError_t launch_argmax_reduce_pair(const float* amax_val, const int* amax_idx, int M, int n_tiles, int idx_offset, void* pair_out,
                                      cudaStream_t s);
cudaError_t launch_ar_argmax(void* const* d_peer_arg, int t, int M, int32_t* out_ids, cudaStream_t s);

}  // namespace oa
