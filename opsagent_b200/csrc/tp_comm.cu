// tp_comm.cu — see tp_comm.hpp.  Cross-GPU all-reduce over NVLink peer memory with the engine's own kernels.
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <signal.h>
#include <cerrno>

#include <chrono>
#include <cstdio>
#include <cstring>
#include <functional>
#include <stdexcept>
#include <thread>

#include "common.cuh"
#include "model.hpp"
#include "tp_comm.hpp"
#include "sk_consumers.cuh"

namespace oa {

static void spin_until(const std::function<bool()>& ok, const char* what, double timeout_s = 120.0) {
    const auto t0 = std::chrono::steady_clock::now();
    while (!ok()) {
        std::this_thread::sleep_for(std::chrono::microseconds(200));
        if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > timeout_s)
            throw std::runtime_error(std::string("tensor-parallel rendezvous timed out: ") + what);
    }
}

static bool pid_alive(int64_t pid) { return pid > 0 && (kill((pid_t)pid, 0) == 0 || errno != ESRCH); }

TpComm::TpComm(int t, int rank, const std::string& shm_name, size_t sym_bytes, int max_sample, uint64_t nonce, size_t nvls_bytes)
    : t_(t), rank_(rank), shm_name_(shm_name), sym_bytes_(sym_bytes) {
    if (t < 2 || t > TP_MAX || rank < 0 || rank >= t) throw std::runtime_error("tp must be 2..8 and 0 <= tp_rank < tp");
    // ---- shared-memory segment (leader creates, followers attach) ----
    // A crashed run leaves its segment behind with magic set, handles_ready >= t and possibly seq == UINT64_MAX.  The new leader therefore
    // first INVALIDATES whatever is linked under the name (magic = 0: a follower that attached to it goes back to waiting), then unlinks
    // and creates a fresh segment stamped with this launch's nonce and its own pid; followers accept a segment only if the nonce matches
    // theirs (when one is configured) and the leader process is alive, and otherwise keep polling for the new one.
    if (rank == 0) {
        int old = shm_open(shm_name.c_str(), O_RDWR, 0600);
        if (old >= 0) {
            struct stat st;
            if (fstat(old, &st) == 0 && (size_t)st.st_size >= sizeof(TpShm)) {
                void* m = mmap(nullptr, sizeof(TpShm), PROT_READ | PROT_WRITE, MAP_SHARED, old, 0);
                if (m != MAP_FAILED) {
                    TpShm* stale = reinterpret_cast<TpShm*>(m);
                    const int64_t owner = stale->leader_pid.load();
                    if (stale->magic.load() == 0x4f415450u && owner != (int64_t)getpid() && pid_alive(owner) && stale->seq.load() != UINT64_MAX) {
                        munmap(m, sizeof(TpShm)); close(old);
                        throw std::runtime_error("tp shm segment " + shm_name + " belongs to a live tensor-parallel group (leader pid " + std::to_string((long long)owner) +
                                                 "): give this group its own \"tp_shm\" name");
                    }
                    stale->magic.store(0, std::memory_order_release);
                    munmap(m, sizeof(TpShm));
                }
            }
            close(old);
        }
        shm_unlink(shm_name.c_str());
        const int fd = shm_open(shm_name.c_str(), O_CREAT | O_EXCL | O_RDWR, 0600);
        if (fd < 0 || ftruncate(fd, sizeof(TpShm)) != 0) throw std::runtime_error("shm_open/ftruncate failed for " + shm_name);
        owner_ = true;
        shm_ = reinterpret_cast<TpShm*>(mmap(nullptr, sizeof(TpShm), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0));
        close(fd);
        if (shm_ == MAP_FAILED) throw std::runtime_error("mmap of the tp shm segment failed");
        shm_->handles_ready.store(0); shm_->peers_opened.store(0); shm_->seq.store(0);
        for (int i = 0; i < TP_MAX; ++i) shm_->ack[i].store(0);
        for (int i = 0; i < TP_MAX; ++i) shm_->rank_pid[i].store(0);
        shm_->nvls_leader_ready.store(0); shm_->nvls_stage[0].store(0); shm_->nvls_stage[1].store(0); shm_->nvls_fail.store(0);
        shm_->nonce.store(nonce); shm_->leader_pid.store((int64_t)getpid());
        shm_->magic.store(0x4f415450u, std::memory_order_release);
    } else {
        spin_until([&] {
            const int fd = shm_open(shm_name.c_str(), O_RDWR, 0600); if (fd < 0) return false;
            struct stat st; if (fstat(fd, &st) != 0 || (size_t)st.st_size < sizeof(TpShm)) { close(fd); return false; }
            void* m = mmap(nullptr, sizeof(TpShm), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
            close(fd);
            if (m == MAP_FAILED) return false;
            TpShm* c = reinterpret_cast<TpShm*>(m);
            const bool ok = c->magic.load(std::memory_order_acquire) == 0x4f415450u && (nonce == 0 || c->nonce.load() == nonce) &&
                            pid_alive(c->leader_pid.load()) && c->seq.load() != UINT64_MAX;
            if (!ok) { munmap(m, sizeof(TpShm)); return false; }      // not there yet, stale, or another launch's: keep polling
            shm_ = c; return true; },
                   "follower waiting for the leader's shm segment (same tp_shm name and tp_nonce, live leader)");
    }
    shm_->rank_pid[rank].store((int64_t)getpid());
    // ---- symmetric device buffers + IPC handle exchange ----
    arg_half_bytes_ = (size_t)max_sample * 8;
    for (int b = 0; b < 3; ++b) { cuda_check(cudaMalloc(&sym_[b], sym_bytes), "cudaMalloc sym"); cuda_check(cudaMemset(sym_[b], 0, sym_bytes), "memset sym"); }
    cuda_check(cudaMalloc(reinterpret_cast<void**>(&flags_), TP_MAX * sizeof(uint32_t)), "cudaMalloc flags");
    cuda_check(cudaMemset(flags_, 0, TP_MAX * sizeof(uint32_t)), "memset flags");
    cuda_check(cudaMalloc(reinterpret_cast<void**>(&done_counter_), 64), "cudaMalloc done counter");
    cuda_check(cudaMemset(done_counter_, 0, 64), "memset done counter");
    cuda_check(cudaMalloc(&arg_, 2 * arg_half_bytes_), "cudaMalloc arg");
    cuda_check(cudaDeviceSynchronize(), "sync");
    for (int b = 0; b < 3; ++b) cuda_check(cudaIpcGetMemHandle(&shm_->h_sym[rank][b], sym_[b]), "cudaIpcGetMemHandle sym");
    cuda_check(cudaIpcGetMemHandle(&shm_->h_flags[rank], flags_), "cudaIpcGetMemHandle flags");
    cuda_check(cudaIpcGetMemHandle(&shm_->h_arg[rank], arg_), "cudaIpcGetMemHandle arg");
    shm_->handles_ready.fetch_add(1, std::memory_order_acq_rel);
    spin_until([&] { return shm_->handles_ready.load(std::memory_order_acquire) >= (uint32_t)t; }, "all ranks publishing IPC handles");
    for (int p = 0; p < t; ++p) {
        if (p == rank) { peer_sym_[0][p] = sym_[0]; peer_sym_[1][p] = sym_[1]; peer_sym_[2][p] = sym_[2]; peer_flags_[p] = flags_; peer_arg_[p] = arg_; continue; }
        for (int b = 0; b < 3; ++b) cuda_check(cudaIpcOpenMemHandle(&peer_sym_[b][p], shm_->h_sym[p][b], cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle sym");
        cuda_check(cudaIpcOpenMemHandle(reinterpret_cast<void**>(&peer_flags_[p]), shm_->h_flags[p], cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle flags");
        cuda_check(cudaIpcOpenMemHandle(&peer_arg_[p], shm_->h_arg[p], cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle arg");
    }
    cuda_check(cudaMalloc(reinterpret_cast<void**>(&d_peer_sym_[2]), TP_MAX * sizeof(void*)), "cudaMalloc ptr table");
    cuda_check(cudaMemcpy(d_peer_sym_[2], peer_sym_[2], TP_MAX * sizeof(void*), cudaMemcpyHostToDevice), "ptr table H2D");
    for (int b = 0; b < 2; ++b) {
        cuda_check(cudaMalloc(reinterpret_cast<void**>(&d_peer_sym_[b]), TP_MAX * sizeof(void*)), "cudaMalloc ptr table");
        cuda_check(cudaMemcpy(d_peer_sym_[b], peer_sym_[b], TP_MAX * sizeof(void*), cudaMemcpyHostToDevice), "ptr table H2D");
        void* pa[TP_MAX] = {};
        for (int p = 0; p < t; ++p) pa[p] = reinterpret_cast<char*>(peer_arg_[p]) + (size_t)b * arg_half_bytes_;
        cuda_check(cudaMalloc(reinterpret_cast<void**>(&d_peer_arg_[b]), TP_MAX * sizeof(void*)), "cudaMalloc ptr table");
        cuda_check(cudaMemcpy(d_peer_arg_[b], pa, TP_MAX * sizeof(void*), cudaMemcpyHostToDevice), "ptr table H2D");
    }
    cuda_check(cudaMalloc(reinterpret_cast<void**>(&d_peer_flags_), TP_MAX * sizeof(uint32_t*)), "cudaMalloc ptr table");
    cuda_check(cudaMemcpy(d_peer_flags_, peer_flags_, TP_MAX * sizeof(uint32_t*), cudaMemcpyHostToDevice), "ptr table H2D");
    shm_->peers_opened.fetch_add(1, std::memory_order_acq_rel);
    spin_until([&] { return shm_->peers_opened.load(std::memory_order_acquire) >= (uint32_t)t; }, "all ranks mapping their peers");
    if (nvls_bytes > 0) nvls_setup(nvls_bytes, nonce);          // all ranks or none (tp_nvls.cpp); failure only means the peer-memory path stays
}

TpComm::~TpComm() {
    nvls_teardown();
    for (int p = 0; p < t_; ++p) {
        if (p == rank_) continue;
        for (int b = 0; b < 3; ++b) if (peer_sym_[b][p]) cudaIpcCloseMemHandle(peer_sym_[b][p]);
        if (peer_flags_[p]) cudaIpcCloseMemHandle(peer_flags_[p]);
        if (peer_arg_[p]) cudaIpcCloseMemHandle(peer_arg_[p]);
    }
    for (int b = 0; b < 2; ++b) { cudaFree(sym_[b]); cudaFree(d_peer_sym_[b]); cudaFree(d_peer_arg_[b]); }
    cudaFree(sym_[2]); cudaFree(d_peer_sym_[2]);
    cudaFree(flags_); cudaFree(arg_); cudaFree(d_peer_flags_); cudaFree(done_counter_);
    if (shm_ && shm_ != MAP_FAILED) munmap(shm_, sizeof(TpShm));
    if (owner_) shm_unlink(shm_name_.c_str());
}

// ---------------------------------------------------------------------------------------------
// host-side step broadcast
// ---------------------------------------------------------------------------------------------
void TpComm::publish(const StepInput& in) {
    // the previous message must have been consumed by every follower before it is overwritten
    const uint64_t cur = shm_->seq.load(std::memory_order_acquire);
    for (int p = 1; p < t_; ++p) {
        uint64_t polls = 0;
        spin_until([&] {
            if (shm_->ack[p].load(std::memory_order_acquire) >= cur) return true;
            if ((++polls & 0x7ff) == 0 && !pid_alive(shm_->rank_pid[p].load()))      // every ~0.4 s
                throw std::runtime_error("tensor-parallel follower " + std::to_string(p) + " (pid " + std::to_string((long long)shm_->rank_pid[p].load()) + ") is gone");
            return false; }, "followers acknowledging the previous step", 600.0);
    }
    int32_t* m = shm_->msg; size_t w = 0;
    auto put = [&](const void* src, size_t words) { if (w + words > TP_MSG_WORDS) throw std::runtime_error("tp step message overflow"); std::memcpy(m + w, src, words * 4); w += words; };
    const int32_t hdr[10] = {(in.decode ? 1 : 0) | (in.n_decode << 1), (int32_t)in.tokens.size(), (int32_t)in.sample_rows.size(), in.n_seqs, (int32_t)in.block_tables.size(),
                             (int32_t)in.ctx_lens.size(), (int32_t)in.tiles.size(), (in.want_logits ? 1 : 0), (int32_t)in.mask_slots.size(), (int32_t)in.mask_updates.size()};
    put(hdr, 10);
    put(in.tokens.data(), in.tokens.size()); put(in.positions.data(), in.positions.size()); put(in.slots.data(), in.slots.size());
    put(in.sample_rows.data(), in.sample_rows.size()); put(in.block_tables.data(), in.block_tables.size());
    put(in.ctx_lens.data(), in.ctx_lens.size()); put(in.tiles.data(), in.tiles.size() * 4); put(in.mask_slots.data(), in.mask_slots.size()); put(in.mask_updates.data(), in.mask_updates.size());
    shm_->msg_words = (uint32_t)w;
    shm_->seq.store(cur + 1, std::memory_order_release);
}

bool TpComm::receive(StepInput& in) {
    uint64_t s = 0;
    while (true) {
        s = shm_->seq.load(std::memory_order_acquire);
        if (s == UINT64_MAX) return false;
        if (s > seq_local_) break;
        std::this_thread::sleep_for(std::chrono::microseconds(20));
        if ((++idle_polls_ & 0x3fff) == 0 && !leader_alive())      // every ~0.3 s of idling
            throw std::runtime_error("tensor-parallel leader (pid " + std::to_string((long long)shm_->leader_pid.load()) + ") is gone");
    }
    const int32_t* m = shm_->msg; size_t w = 0;
    const int32_t* hdr = m; w += 10;
    auto get = [&](std::vector<int32_t>& v, int n) { v.assign(m + w, m + w + n); w += n; };
    in = StepInput();
    in.decode = (hdr[0] & 1) != 0; in.n_decode = hdr[0] >> 1; in.n_seqs = hdr[3]; in.want_logits = (hdr[7] & 1) != 0;
    get(in.tokens, hdr[1]); get(in.positions, hdr[1]); get(in.slots, hdr[1]); get(in.sample_rows, hdr[2]);
    get(in.block_tables, hdr[4]); get(in.ctx_lens, hdr[5]);
    in.tiles.resize(hdr[6]); std::memcpy(in.tiles.data(), m + w, (size_t)hdr[6] * 16); w += (size_t)hdr[6] * 4;
    get(in.mask_slots, hdr[8]);
    in.mask_updates.resize((size_t)hdr[9]); std::memcpy(in.mask_updates.data(), m + w, (size_t)hdr[9] * 4); w += (size_t)hdr[9];
    seq_local_ = s;
    shm_->ack[rank_].store(s, std::memory_order_release);
    return true;
}

bool TpComm::leader_alive() const { return shm_ && pid_alive(shm_->leader_pid.load()); }

void TpComm::shutdown() { if (shm_ && rank_ == 0) shm_->seq.store(UINT64_MAX, std::memory_order_release); }

// ---------------------------------------------------------------------------------------------
// device side
// ---------------------------------------------------------------------------------------------
OA_DEVINL void st_release_sys(uint32_t* p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
OA_DEVINL uint32_t ld_acquire_sys(const uint32_t* p) { uint32_t v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
OA_DEVINL float4 ld_peer_f4(const float* p) { float4 v; asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p)); return v; }
OA_DEVINL uint4 ld_peer_u4(const void* p) { uint4 v; asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)); return v; }

// Thread p tells peer p "rank `rank` has finished everything before epoch e" and waits for peer p's matching flag.
__global__ void xgpu_barrier_kernel(uint32_t* const* __restrict__ peer_flags, const uint32_t* __restrict__ my_flags, int rank, int t, uint32_t epoch) {
    griddep_launch(); griddep_wait();
    const int p = threadIdx.x;
    if (p < t) {
        __threadfence_system();
        st_release_sys(peer_flags[p] + rank, epoch);
        const long long t0 = clock64();
        while ((int32_t)(ld_acquire_sys(my_flags + p) - epoch) < 0) {
            if (clock64() - t0 > (long long)3.0e10) __trap();          // ~15 s: a peer died
        }
    }
}
cudaError_t TpComm::barrier(cudaStream_t s) {
    ++epoch_;
    return launch_k(xgpu_barrier_kernel, dim3(1), dim3(32), 0, s, (uint32_t* const*)d_peer_flags_, (const uint32_t*)flags_, rank_, t_, epoch_);
}

// producer side of the split handshake: called by every thread of every CTA after its last store to the symmetric buffer
OA_DEVINL void xgpu_signal_when_grid_done(const TpComm::Signal& sg, unsigned int n_ctas) {
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int old = atomicAdd(sg.done_counter, 1u);
        s_last = old == n_ctas - 1u;
        if (s_last) *sg.done_counter = 0u;            // re-arm for the next collective
    }
    __syncthreads();
    if (s_last && (int)threadIdx.x < sg.t) {
        __threadfence_system();
        st_release_sys(sg.peer_flags[threadIdx.x] + sg.rank, sg.epoch);
    }
}
// consumer side: wait until every peer has signalled `epoch`
OA_DEVINL void xgpu_wait_peers(const TpComm::Signal& sg) {
    if ((int)threadIdx.x < sg.t) {
        const long long t0 = clock64();
        while ((int32_t)(ld_acquire_sys(sg.my_flags + threadIdx.x) - sg.epoch) < 0) {
            if (clock64() - t0 > (long long)3.0e10) __trap();          // ~15 s: a peer died
        }
    }
    __syncthreads();
}

// One CTA per token row, 1024 threads, 16-byte items: lane l of a warp loads bytes [16l, 16l+16) of a 512-byte run, so every
// peer load instruction is four full 128-byte lines on the NVLink (32-byte items at a 32-byte stride were half-used sectors).
constexpr int AR_THREADS = 1024;
__global__ void __launch_bounds__(AR_THREADS) ar_resid_rmsnorm_kernel(const float* const* __restrict__ peer, int t, uint2* __restrict__ x,
                                                                      const uint2* __restrict__ g, uint2* __restrict__ y, int H4, float inv_h, float eps,
                                                                      const TpComm::Signal sg, int wait) {
    griddep_launch(); griddep_wait();
    if (wait) xgpu_wait_peers(sg);
    const int row = blockIdx.x;
    uint2* xr = x + (size_t)row * H4;
    float ss = 0.f;
    for (int i = threadIdx.x; i < H4; i += AR_THREADS) {
        float4 a[TP_MAX];
#pragma unroll
        for (int p = 0; p < TP_MAX; ++p) if (p < t) a[p] = ld_peer_f4(peer[p] + ((size_t)row * H4 + i) * 4);
        const uint2 xo = xr[i];
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int p = 0; p < TP_MAX; ++p) if (p < t) { acc[0] += a[p].x; acc[1] += a[p].y; acc[2] += a[p].z; acc[3] += a[p].w; }   // rank order: identical on every rank
        uint2 xn;
        xn.x = pack_bf16x2(bf16lo(xo.x) + acc[0], bf16hi(xo.x) + acc[1]); xn.y = pack_bf16x2(bf16lo(xo.y) + acc[2], bf16hi(xo.y) + acc[3]);
        xr[i] = xn;
        float q;
        q = bf16lo(xn.x); ss += q * q; q = bf16hi(xn.x); ss += q * q; q = bf16lo(xn.y); ss += q * q; q = bf16hi(xn.y); ss += q * q;
    }
    ss = warp_sum(ss);
    __shared__ float red[AR_THREADS / 32];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < AR_THREADS / 32; ++w) tot += red[w];
    const float r = 1.0f / sqrtf(tot * inv_h + eps);
    uint2* yr = y + (size_t)row * H4;
    for (int i = threadIdx.x; i < H4; i += AR_THREADS) {      // this thread re-reads exactly what it wrote above
        const uint2 v = xr[i], gg = g[i]; uint2 o;
        o.x = pack_bf16x2(bf16lo(v.x) * r * bf16lo(gg.x), bf16hi(v.x) * r * bf16hi(gg.x));
        o.y = pack_bf16x2(bf16lo(v.y) * r * bf16lo(gg.y), bf16hi(v.y) * r * bf16hi(gg.y));
        yr[i] = o;
    }
}
cudaError_t launch_ar_resid_rmsnorm(void* const* d_peer, int t, void* x, const void* gain, void* xn, int T, int H, float eps, cudaStream_t s,
                                    const TpComm::Signal* wait) {
    if (T <= 0) return cudaSuccess;
    if (H % 8 != 0) return cudaErrorInvalidValue;
    auto P = reinterpret_cast<const float* const*>(d_peer);
    const TpComm::Signal sg = wait ? *wait : TpComm::Signal{};
    return launch_k(ar_resid_rmsnorm_kernel, dim3(T), dim3(AR_THREADS), 0, s, P, t, reinterpret_cast<uint2*>(x), reinterpret_cast<const uint2*>(gain),
                    reinterpret_cast<uint2*>(xn), H / 4, 1.0f / H, eps, sg, wait ? 1 : 0);
}

// ---- in-switch all-reduce (NVLS multicast, tp_nvls.cpp) -------------------------------------------------------------------------
OA_DEVINL float4 multimem_ld_reduce_f4(const float* mc) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
    return v;
}
OA_DEVINL void multimem_st_f4(float* mc, const float4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
OA_DEVINL void multimem_st_release_u32(uint32_t* mc, uint32_t v) { asm volatile("multimem.st.release.sys.global.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory"); }
// One CTA per token row.  Row c is OWNED by rank c % t: the owner's CTA asks the switch for the sum of the row over all ranks and broadcasts it,
// then broadcasts the row's flag (multimem.st.release after a system fence); every rank's CTA c waits for exactly that one flag in its local copy
// and finishes residual + RMSNorm from local memory.  No grid-wide barrier and no all-to-all handshake in the middle: the only cross-GPU
// round trips are the owner's ld_reduce and its two broadcasts.
__global__ void __launch_bounds__(AR_THREADS) ar_nvls_resid_rmsnorm_kernel(const float* __restrict__ mc_part, float* __restrict__ mc_red, const float* __restrict__ local_red,
                                                                           uint32_t* __restrict__ mc_flags, const uint32_t* __restrict__ local_flags,
                                                                           int t, int rank, uint2* __restrict__ x, const uint2* __restrict__ g, uint2* __restrict__ y,
                                                                           int H4, float inv_h, float eps, const TpComm::Signal sg_in, uint32_t epoch) {
    griddep_wait();
    const int row = blockIdx.x;
    if (row % t == rank) {
        xgpu_wait_peers(sg_in);                               // every rank's partial is complete in its copy of the buffer
        for (int i = threadIdx.x; i < H4; i += AR_THREADS) {
            const float4 v = multimem_ld_reduce_f4(mc_part + ((size_t)row * H4 + i) * 4);
            multimem_st_f4(mc_red + ((size_t)row * H4 + i) * 4, v);
        }
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) { __threadfence_system(); multimem_st_release_u32(mc_flags + row, epoch); }
    }
    if (threadIdx.x == 0) {
        const long long t0 = clock64();
        while ((int32_t)(ld_acquire_sys(local_flags + row) - epoch) < 0) {
            if (clock64() - t0 > (long long)3.0e10) __trap();          // ~15 s: the row's owner died
        }
    }
    __syncthreads();
    griddep_launch();
    uint2* xr = x + (size_t)row * H4;
    float ss = 0.f;
    for (int i = threadIdx.x; i < H4; i += AR_THREADS) {
        const float4 a = __ldcg(reinterpret_cast<const float4*>(local_red) + (size_t)row * H4 + i);      // written by a multicast store: bypass L1
        const uint2 xo = xr[i];
        uint2 xn;
        xn.x = pack_bf16x2(bf16lo(xo.x) + a.x, bf16hi(xo.x) + a.y); xn.y = pack_bf16x2(bf16lo(xo.y) + a.z, bf16hi(xo.y) + a.w);
        xr[i] = xn;
        float q;
        q = bf16lo(xn.x); ss += q * q; q = bf16hi(xn.x); ss += q * q; q = bf16lo(xn.y); ss += q * q; q = bf16hi(xn.y); ss += q * q;
    }
    ss = warp_sum(ss);
    __shared__ float red[AR_THREADS / 32];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < AR_THREADS / 32; ++w) tot += red[w];
    const float r = 1.0f / sqrtf(tot * inv_h + eps);
    uint2* yr = y + (size_t)row * H4;
    for (int i = threadIdx.x; i < H4; i += AR_THREADS) {
        const uint2 v = xr[i], gg = g[i]; uint2 o;
        o.x = pack_bf16x2(bf16lo(v.x) * r * bf16lo(gg.x), bf16hi(v.x) * r * bf16hi(gg.x));
        o.y = pack_bf16x2(bf16lo(v.y) * r * bf16lo(gg.y), bf16hi(v.y) * r * bf16hi(gg.y));
        yr[i] = o;
    }
}
cudaError_t launch_ar_nvls_resid_rmsnorm(const void* mc_base, const void* local_base, size_t part_off, size_t red_off, size_t flag_off, int t, int rank, void* x,
                                         const void* gain, void* xn, int T, int H, float eps, cudaStream_t s, const TpComm::Signal& wait) {
    if (T <= 0) return cudaSuccess;
    if (H % 8 != 0 || T > 132) return cudaErrorInvalidValue;            // CTAs wait for flags set by other ranks' CTAs of the same launch: keep the grid co-resident
    char* mc = reinterpret_cast<char*>(const_cast<void*>(mc_base)); const char* lc = reinterpret_cast<const char*>(local_base);
    return launch_k(ar_nvls_resid_rmsnorm_kernel, dim3(T), dim3(AR_THREADS), 0, s, reinterpret_cast<const float*>(mc + part_off), reinterpret_cast<float*>(mc + red_off),
                    reinterpret_cast<const float*>(lc + red_off), reinterpret_cast<uint32_t*>(mc + flag_off), reinterpret_cast<const uint32_t*>(lc + flag_off), t, rank,
                    reinterpret_cast<uint2*>(x), reinterpret_cast<const uint2*>(gain), reinterpret_cast<uint2*>(xn), H / 4, 1.0f / H, eps, wait, wait.epoch);
}

// The same collective on bf16 partials: half the NVLink bytes (the one-shot all-reduce of a decode step is bandwidth-bound: every rank
// reads t full partials — 70B TP=8, B=64: 16.8 MB in fp32).  Each rank rounds its fp32 partial to bf16 once (as the prefill path's tile
// GEMM always did), the sum over ranks is fp32 in rank order, so all ranks still hold bit-identical activations.
__global__ void __launch_bounds__(AR_THREADS) ar_resid_rmsnorm_bf16in_kernel(const uint16_t* const* __restrict__ peer, int t, uint4* __restrict__ x,
                                                                             const uint4* __restrict__ g, uint4* __restrict__ y, int H8, float inv_h, float eps,
                                                                             const TpComm::Signal sg, int wait) {
    griddep_launch(); griddep_wait();
    if (wait) xgpu_wait_peers(sg);
    const int row = blockIdx.x;
    uint4* xr = x + (size_t)row * H8;
    float ss = 0.f;
    for (int i = threadIdx.x; i < H8; i += AR_THREADS) {
        uint4 a[TP_MAX];
#pragma unroll
        for (int p = 0; p < TP_MAX; ++p) if (p < t) a[p] = ld_peer_u4(peer[p] + ((size_t)row * H8 + i) * 8);
        const uint4 xo = xr[i];
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int p = 0; p < TP_MAX; ++p) if (p < t) {      // rank order: identical on every rank
            acc[0] += bf16lo(a[p].x); acc[1] += bf16hi(a[p].x); acc[2] += bf16lo(a[p].y); acc[3] += bf16hi(a[p].y);
            acc[4] += bf16lo(a[p].z); acc[5] += bf16hi(a[p].z); acc[6] += bf16lo(a[p].w); acc[7] += bf16hi(a[p].w);
        }
        uint4 xn;
        xn.x = pack_bf16x2(bf16lo(xo.x) + acc[0], bf16hi(xo.x) + acc[1]); xn.y = pack_bf16x2(bf16lo(xo.y) + acc[2], bf16hi(xo.y) + acc[3]);
        xn.z = pack_bf16x2(bf16lo(xo.z) + acc[4], bf16hi(xo.z) + acc[5]); xn.w = pack_bf16x2(bf16lo(xo.w) + acc[6], bf16hi(xo.w) + acc[7]);
        xr[i] = xn;
        float q;
        q = bf16lo(xn.x); ss += q * q; q = bf16hi(xn.x); ss += q * q; q = bf16lo(xn.y); ss += q * q; q = bf16hi(xn.y); ss += q * q;
        q = bf16lo(xn.z); ss += q * q; q = bf16hi(xn.z); ss += q * q; q = bf16lo(xn.w); ss += q * q; q = bf16hi(xn.w); ss += q * q;
    }
    ss = warp_sum(ss);
    __shared__ float red[AR_THREADS / 32];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < AR_THREADS / 32; ++w) tot += red[w];
    const float r = 1.0f / sqrtf(tot * inv_h + eps);
    uint4* yr = y + (size_t)row * H8;
    for (int i = threadIdx.x; i < H8; i += AR_THREADS) {      // this thread re-reads exactly what it wrote above
        const uint4 v = xr[i], gg = g[i]; uint4 o;
        o.x = pack_bf16x2(bf16lo(v.x) * r * bf16lo(gg.x), bf16hi(v.x) * r * bf16hi(gg.x));
        o.y = pack_bf16x2(bf16lo(v.y) * r * bf16lo(gg.y), bf16hi(v.y) * r * bf16hi(gg.y));
        o.z = pack_bf16x2(bf16lo(v.z) * r * bf16lo(gg.z), bf16hi(v.z) * r * bf16hi(gg.z));
        o.w = pack_bf16x2(bf16lo(v.w) * r * bf16lo(gg.w), bf16hi(v.w) * r * bf16hi(gg.w));
        yr[i] = o;
    }
}
cudaError_t launch_ar_resid_rmsnorm_bf16in(void* const* d_peer, int t, void* x, const void* gain, void* xn, int T, int H, float eps, cudaStream_t s,
                                           const TpComm::Signal* wait) {
    if (T <= 0) return cudaSuccess;
    if (H % 8 != 0) return cudaErrorInvalidValue;
    const TpComm::Signal sg = wait ? *wait : TpComm::Signal{};
    return launch_k(ar_resid_rmsnorm_bf16in_kernel, dim3(T), dim3(AR_THREADS), 0, s, reinterpret_cast<const uint16_t* const*>(d_peer), t, reinterpret_cast<uint4*>(x),
                    reinterpret_cast<const uint4*>(gain), reinterpret_cast<uint4*>(xn), H / 8, 1.0f / H, eps, sg, wait ? 1 : 0);
}

__global__ void ar_resid_bf16_kernel(const uint16_t* const* __restrict__ peer, int t, uint4* __restrict__ x, size_t n8) {
    griddep_launch(); griddep_wait();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        uint4 a[TP_MAX];
#pragma unroll
        for (int p = 0; p < TP_MAX; ++p) if (p < t) a[p] = ld_peer_u4(peer[p] + i * 8);
#pragma unroll
        for (int p = 0; p < TP_MAX; ++p) if (p < t) {
            acc[0] += bf16lo(a[p].x); acc[1] += bf16hi(a[p].x); acc[2] += bf16lo(a[p].y); acc[3] += bf16hi(a[p].y);
            acc[4] += bf16lo(a[p].z); acc[5] += bf16hi(a[p].z); acc[6] += bf16lo(a[p].w); acc[7] += bf16hi(a[p].w);
        }
        add_bf16x8(acc, x[i]);
        x[i] = pack_bf16x8(acc);
    }
}
cudaError_t launch_ar_resid_bf16(void* const* d_peer, int t, void* x, int T, int H, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    const size_t n8 = (size_t)T * H / 8;
    const int blocks = (int)std::min<size_t>((n8 + 255) / 256, 132 * 8);
    return launch_k(ar_resid_bf16_kernel, dim3(blocks), dim3(256), 0, s, reinterpret_cast<const uint16_t* const*>(d_peer), t, reinterpret_cast<uint4*>(x), n8);
}

// ---- two-shot all-reduce for prefill-sized batches (see tp_comm.hpp) ----
// flat partition of the T*H/8 16-byte vectors into t contiguous slices; slice r belongs to rank r
OA_DEVINL void ar2_slice(size_t n8, int t, int r, size_t& lo, size_t& hi) { const size_t per = (n8 + (size_t)t - 1) / (size_t)t; lo = (size_t)r * per; hi = lo + per < n8 ? lo + per : n8; if (lo > n8) lo = n8; }
__global__ void ar2_reduce_scatter_kernel(const uint16_t* const* __restrict__ peer, int t, int rank, uint4* __restrict__ x, uint4* __restrict__ gather, size_t n8) {
    griddep_launch(); griddep_wait();
    size_t lo, hi; ar2_slice(n8, t, rank, lo, hi);
    for (size_t i = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (size_t)gridDim.x * blockDim.x) {
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        uint4 a[TP_MAX];
#pragma unroll
        for (int p = 0; p < TP_MAX; ++p) if (p < t) a[p] = ld_peer_u4(peer[p] + i * 8);
#pragma unroll
        for (int p = 0; p < TP_MAX; ++p) if (p < t) {      // rank order
            acc[0] += bf16lo(a[p].x); acc[1] += bf16hi(a[p].x); acc[2] += bf16lo(a[p].y); acc[3] += bf16hi(a[p].y);
            acc[4] += bf16lo(a[p].z); acc[5] += bf16hi(a[p].z); acc[6] += bf16lo(a[p].w); acc[7] += bf16hi(a[p].w);
        }
        add_bf16x8(acc, x[i]);
        const uint4 xn = pack_bf16x8(acc);
        x[i] = xn; gather[i] = xn;
    }
}
__global__ void ar2_all_gather_kernel(const uint16_t* const* __restrict__ peer, int t, int rank, uint4* __restrict__ x, size_t n8) {
    griddep_launch(); griddep_wait();
    for (int q = 1; q < t; ++q) {
        const int p = (rank + q) % t;                       // start with the next rank: spreads the first reads over all links
        size_t lo, hi; ar2_slice(n8, t, p, lo, hi);
        for (size_t i = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (size_t)gridDim.x * blockDim.x) x[i] = ld_peer_u4(peer[p] + i * 8);
    }
}
cudaError_t launch_ar2_reduce_scatter(void* const* d_peer_partial, int t, int rank, void* x, void* gather_mine, int T, int H, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    const size_t n8 = (size_t)T * H / 8;
    const int blocks = (int)std::min<size_t>((n8 / t + 255) / 256 + 1, 132 * 8);
    return launch_k(ar2_reduce_scatter_kernel, dim3(blocks), dim3(256), 0, s, reinterpret_cast<const uint16_t* const*>(d_peer_partial), t, rank, reinterpret_cast<uint4*>(x),
                    reinterpret_cast<uint4*>(gather_mine), n8);
}
cudaError_t launch_ar2_all_gather(void* const* d_peer_gather, int t, int rank, void* x, int T, int H, cudaStream_t s) {
    if (T <= 0) return cudaSuccess;
    const size_t n8 = (size_t)T * H / 8;
    const int blocks = (int)std::min<size_t>((n8 / t + 255) / 256 + 1, 132 * 8);
    return launch_k(ar2_all_gather_kernel, dim3(blocks), dim3(256), 0, s, reinterpret_cast<const uint16_t* const*>(d_peer_gather), t, rank, reinterpret_cast<uint4*>(x), n8);
}

__global__ void sk_reduce_f32_rows_kernel(const StreamK sk, float* __restrict__ out, int N8, const TpComm::Signal sg, int signal) {
    griddep_launch(); griddep_wait();
    const int row = blockIdx.y;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N8; i += gridDim.x * blockDim.x) {
        float acc[8];
        sk_sum8(sk, row, i * 8, acc);            // CTA order, up to 6 pieces' loads in flight together
        float4* o = reinterpret_cast<float4*>(out + ((size_t)row * N8 + i) * 8);
        o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]); o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    if (signal) xgpu_signal_when_grid_done(sg, gridDim.x * gridDim.y);
}
cudaError_t launch_sk_reduce_f32(const StreamK& sk, float* out, int T, int N, cudaStream_t s, const TpComm::Signal* signal) {
    if (T <= 0) return cudaSuccess;
    const TpComm::Signal sg = signal ? *signal : TpComm::Signal{};
    return launch_k(sk_reduce_f32_rows_kernel, dim3((N / 8 + 255) / 256, T), dim3(256), 0, s, sk, out, N / 8, sg, signal ? 1 : 0);
}

__global__ void sk_reduce_bf16_rows_kernel(const StreamK sk, uint4* __restrict__ out, int N8, const TpComm::Signal sg, int signal) {
    griddep_launch(); griddep_wait();
    const int row = blockIdx.y;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N8; i += gridDim.x * blockDim.x) {
        float acc[8];
        sk_sum8(sk, row, i * 8, acc);            // CTA order, up to 6 pieces' loads in flight together
        uint4 o;
        o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]); o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
        out[(size_t)row * N8 + i] = o;
    }
    if (signal) xgpu_signal_when_grid_done(sg, gridDim.x * gridDim.y);
}
cudaError_t launch_sk_reduce_bf16(const StreamK& sk, void* out, int T, int N, cudaStream_t s, const TpComm::Signal* signal) {
    if (T <= 0) return cudaSuccess;
    const TpComm::Signal sg = signal ? *signal : TpComm::Signal{};
    return launch_k(sk_reduce_bf16_rows_kernel, dim3((N / 8 + 255) / 256, T), dim3(256), 0, s, sk, reinterpret_cast<uint4*>(out), N / 8, sg, signal ? 1 : 0);
}

struct ValIdx { float v; int i; };
__global__ void argmax_reduce_pair_kernel(const float* __restrict__ val, const int* __restrict__ idx, int n_tiles, int idx_offset, ValIdx* __restrict__ out) {
    griddep_launch(); griddep_wait();
    const int row = blockIdx.x;
    float bv; int bi;
    block_argmax_row(val, idx, row, n_tiles, bv, bi);
    if (threadIdx.x == 0) { out[row].v = bv; out[row].i = (bi == 0x7fffffff ? 0 : bi) + idx_offset; }
}
cudaError_t launch_argmax_reduce_pair(const float* amax_val, const int* amax_idx, int M, int n_tiles, int idx_offset, void* pair_out, cudaStream_t s) {
    return launch_k(argmax_reduce_pair_kernel, dim3(M), dim3(256), 0, s, amax_val, amax_idx, n_tiles, idx_offset, reinterpret_cast<ValIdx*>(pair_out));
}
__global__ void ar_argmax_kernel(const ValIdx* const* __restrict__ peer, int t, int M, int32_t* __restrict__ out_ids) {
    griddep_launch(); griddep_wait();
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= M) return;
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int p = 0; p < t; ++p) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(peer[p] + row);
        uint32_t a, b;
        asm volatile("ld.relaxed.sys.global.v2.u32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "l"(src));
        const float v = __uint_as_float(a); const int i = (int)b;
        if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
    out_ids[row] = bi;
}
cudaError_t launch_ar_argmax(void* const* d_peer_arg, int t, int M, int32_t* out_ids, cudaStream_t s) {
    return launch_k(ar_argmax_kernel, dim3((M + 127) / 128), dim3(128), 0, s, reinterpret_cast<const ValIdx* const*>(d_peer_arg), t, M, out_ids);
}

}  // namespace oa
