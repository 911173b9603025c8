// model.hpp — device-resident model: weights, paged KV pool, activation buffers, TMA descriptors, and the
// forward pass (prefill chunk or decode step) as a fixed sequence of sm_90a kernel launches on one stream.
#pragma once
#include <memory>
#include <string>
#include <vector>

#include "config.hpp"
#include "kernels.hpp"
#include "stages.hpp"
#include "tp_comm.hpp"

namespace oa {

struct WeightMat {
    void* ptr = nullptr; int N = 0, K = 0;
    bool fp8 = false; float* sw = nullptr;      // fp8: ptr holds e4m3 bytes [N, K], sw the fp32 scale of each row (weight_dtype fp8_e4m3)
    CUtensorMap tm[4];            // B-operand maps for BLOCK_N = 32, 64, 128, 256
    const CUtensorMap* map(int bn) const { return &tm[bn == 32 ? 0 : bn == 64 ? 1 : bn == 128 ? 2 : 3]; }
};

// A projection's input: the bf16 activation buffer [max rows, cols] and, with fp8 weights, its e4m3 copy with one fp32 scale per row,
// which the GEMMs read instead (quantised right before each projection)
struct ProjInput {
    void* x = nullptr; CUtensorMap tm; int cols = 0;
    uint8_t* q = nullptr; float* sc = nullptr; CUtensorMap tm8;      // fp8 weights only
    const CUtensorMap* map() const { return q ? &tm8 : &tm; }
    W8Scales w8(const WeightMat& w) const { return q ? W8Scales{sc, w.sw} : W8Scales{}; }
};

struct StepInput {
    bool decode = false;
    int n_decode = 0;                                 // mixed step (decode == false): the first n_decode rows / sequences are decoding sequences
                                                      // (one token each, decode attention); the prefill chunks follow
    std::vector<int32_t> tokens, positions, slots;   // [T]
    std::vector<int32_t> sample_rows;                 // rows whose next token is wanted
    int n_seqs = 0;
    std::vector<int32_t> block_tables;                // [n_seqs, max_pages_per_seq]
    std::vector<int32_t> ctx_lens;                    // [n_seqs] (decode: tokens in cache incl. the new one)
    std::vector<PrefillTile> tiles;                   // prefill only
    // grammar-constrained sampling: mask_slots[i] = row of the device token-mask table applied to sampled row i (-1: unconstrained); empty: no
    // constrained row.  mask_updates = concatenated records {slot, words[mask_words]} to be written into the table before the LM head.
    std::vector<int32_t> mask_slots; std::vector<uint32_t> mask_updates;
    bool want_logits = false;                         // debug: fp32 logits of the sampled rows (tensor-parallel ranks stage their shard)
};

struct DecodePlan {
    std::vector<DecodeSeg> segs; std::vector<int32_t> cta_ptr; std::vector<MergeItem> merges; int n_slots = 0;
};
// contiguous, balanced partition of all (sequence, kv head) page lists over n_ctas CTAs
void build_decode_plan(const int32_t* ctx_lens, int n_seqs, int n_kv, int n_ctas_target, int force_splits, DecodePlan& out);
// the prefill tiles of `n_rows` new rows of sequence `seq` at token-batch row `row0`, the first at position `pos0`
void append_prefill_tiles(std::vector<PrefillTile>& tiles, int seq, int row0, int pos0, int n_rows);
// the order the prefill-attention grid runs its tiles in: heaviest (most visible keys) first
void sort_prefill_tiles(std::vector<PrefillTile>& tiles);
constexpr int W8_MAX_BN = 128;      // fp8 GEMM tiles are at most 128 wide (registers)
// BLOCK_N of a tile-path GEMM [M, N] on sm_count SMs (override_bn in {32, 64, 128, 256} wins); fp8 operands cap it at W8_MAX_BN
int pick_bn(int M, int N, int sm_count, int override_bn, bool fp8 = false);

class DeviceModel {
public:
    DeviceModel(const ModelConfig& cfg, const EngineOptions& opt);
    ~DeviceModel();
    DeviceModel(const DeviceModel&) = delete;

    // Runs one forward.  Greedy next-token ids of sample_rows land in h_out_ids (pinned) once the stream is
    // synchronised.  logits_out (device fp32 [n_sample, vocab]) is optional.
    void forward(const StepInput& in, float* logits_out);
    void sync();
    // after a completed single-GPU forward with S sampled rows: out[r] = the fp32 logit of the token row r sampled (its LM-head row maximum)
    void sampled_logits(int S, float* out);
    int32_t* h_out_ids = nullptr;        // pinned, [max_batch or max_step_tokens]

    ModelConfig cfg; EngineOptions opt;
    // tensor-parallel shard sizes (== the global sizes when tp == 1)
    int tp = 1, tp_rank = 0, nh_l = 0, nkv_l = 0, F_l = 0, V_l = 0;
    std::unique_ptr<TpComm> comm;
    cudaStream_t stream = nullptr;
    int num_pages = 0, max_pages_per_seq = 0, sm_count = 132;
    int mask_words = 0, mask_slots = 0, max_mask_updates = 0;    // token-mask table geometry (words = ceil(vocab / 32))
    size_t weight_bytes = 0, kv_pool_bytes = 0;
    KvLayout kv{}; CUtensorMap tm_kv;
    std::vector<float> kv_k_scale, kv_v_scale;      // per layer (fp8 cache: from the checkpoint, else 1.0)
    // instrumentation
    bool profile_attn = false; double attn_ms_accum = 0; std::vector<cudaEvent_t> ev;
    // in-situ per-kernel timing (events after every launch, warm caches, real launch gaps): OA_PROFILE_ALL=1
    bool profile_all = false; std::vector<cudaEvent_t> ev_all; std::vector<int> ev_ids; double kt_ms[16] = {0}; long kt_n[16] = {0};
    static const char* kt_name(int id);
    uint64_t h2d_bytes = 0, d2h_bytes = 0;

    struct Layer { WeightMat qkv, o, gu, down; void *ln1 = nullptr, *ln2 = nullptr, *bqkv = nullptr; };
    std::vector<Layer> layers;
    void* embed = nullptr; void* final_norm = nullptr; WeightMat lm_head;
    float *rope_cos = nullptr, *rope_sin = nullptr;

private:
    void alloc_weight(WeightMat& w, int N, int K, bool fp8 = false);
    // a projection weight is written as bf16 [N, K] to bf16_dst(w) (fp8: the shared scratch), then commit(w) quantises an fp8 one into its
    // bytes and row scales (row rule)
    uint16_t* bf16_dst(const WeightMat& w) const { return reinterpret_cast<uint16_t*>(w.fp8 ? w8_scratch_ : w.ptr); }
    void commit(WeightMat& w);
    void load_checkpoint(const std::string& path);     // overwrite the seeded tensors with this rank's slices of an HF checkpoint
    void make_weight_maps(WeightMat& w);
    void* dmalloc(size_t bytes);
    std::vector<void*> allocs_;
    // activations
    void *x_ = nullptr, *qkv_ = nullptr, *q_ = nullptr, *xs_ = nullptr, *xsn_ = nullptr;
    ProjInput xn_, attn_, act_;                    // inputs of qkv and gate/up, of o, of down
    CUtensorMap tm_xsn_;
    void* w8_scratch_ = nullptr;                   // bf16 staging of one projection while the weights are generated or loaded (then freed)
    float* amax_val_ = nullptr; int* amax_idx_ = nullptr; int32_t* d_out_ids_ = nullptr;
    uint32_t* mask_table_ = nullptr;               // [mask_slots][mask_words] allowed-token bitsets of grammar states (filled on demand by the scheduler)
    float *part_o_ = nullptr, *part_ml_ = nullptr; int max_part_slots_ = 0;
    float* sk_ws_ = nullptr; int sk_bn_ = 256, sk_G_ = 132;
    size_t nvls_region_ = 0;                       // bytes of one [128 rows, H] fp32 region of the NVLS multicast buffer (partials 0/1, reduced 0/1)
    unsigned int* tile_flags_ = nullptr;           // per-tile piece counters of the fused stream-K epilogues, [4 projections][SK_MAX_FLAG_TILES] (self-resetting)
    // pinned staging is double-buffered and fenced by events: the host may run ahead of the stream by a whole forward
    int32_t* h_meta_buf_[2] = {nullptr, nullptr}; cudaEvent_t meta_ev_[2] = {nullptr, nullptr}; int meta_idx_ = 0;
    int32_t *h_meta_ = nullptr, *d_meta_ = nullptr; size_t meta_cap_words_ = 0;
    int max_rows_ = 0, max_sample_ = 0;
    DecodePlan plan_; std::vector<int32_t> zero_counters_; std::vector<PrefillTile> sorted_tiles_;
};

}  // namespace oa
