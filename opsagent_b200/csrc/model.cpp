// model.cpp — see model.hpp.
#include "model.hpp"
#include "checkpoint.hpp"

#include <algorithm>
#include <cmath>
#include "common.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

namespace oa {

static void tmap_check(int r, const char* what) {
    if (r != 0) throw std::runtime_error(std::string("cuTensorMapEncodeTiled failed for ") + what + " (code " + std::to_string(r) + ")");
}

// tensor ids of the seeded generator: layer*16 + kind; globals at layer index n_layers (oracle/llama_ref.c)
enum { T_WQ = 0, T_WK, T_WV, T_WO, T_WG, T_WU, T_WD, T_LN1, T_LN2, T_BQ, T_BK, T_BV };
enum { TG_EMBED = 0, TG_NORM = 1, TG_LMHEAD = 2 };

void* DeviceModel::dmalloc(size_t bytes) {
    void* p = nullptr;
    cuda_check(cudaMalloc(&p, bytes ? bytes : 16), "cudaMalloc");
    allocs_.push_back(p);
    return p;
}

void DeviceModel::make_weight_maps(WeightMat& w) {
    const int bns[4] = {32, 64, 128, 256};
    for (int i = 0; i < 4; ++i) {
        tmap_check(w.fp8 ? make_tmap_u8_2d(&w.tm[i], w.ptr, (uint64_t)w.N, (uint64_t)w.K, (uint32_t)bns[i], 128)
                         : make_tmap_bf16_2d(&w.tm[i], w.ptr, (uint64_t)w.N, (uint64_t)w.K, (uint64_t)w.K, (uint32_t)bns[i], 64), "a weight matrix");
    }
}
void DeviceModel::alloc_weight(WeightMat& w, int N, int K, bool fp8) {
    w.N = N; w.K = K; w.fp8 = fp8;
    if (fp8) {
        w.ptr = dmalloc((size_t)N * K); w.sw = reinterpret_cast<float*>(dmalloc((size_t)N * 4)); weight_bytes += (size_t)N * K + (size_t)N * 4;
    } else {
        w.ptr = dmalloc((size_t)N * K * 2); weight_bytes += (size_t)N * K * 2;
    }
    make_weight_maps(w);
}
void DeviceModel::commit(WeightMat& w) {
    if (w.fp8) cuda_check(launch_quant_rows_e4m3(w8_scratch_, reinterpret_cast<uint8_t*>(w.ptr), w.sw, w.N, w.K, stream), "quantise weights (fp8)");
}

// Build the RoPE table exactly as oracle/llama_ref.c:oa_ref_rope_table does (double math, then cast).
static void rope_table(const ModelConfig& c, int max_pos, std::vector<float>& cosv, std::vector<float>& sinv) {
    const int half = c.head_dim / 2;
    cosv.resize((size_t)max_pos * half); sinv.resize((size_t)max_pos * half);
    for (int i = 0; i < half; ++i) {
        double inv = std::pow((double)c.rope_theta, -2.0 * i / (double)c.head_dim);
        if (c.rope_scaling == 1) {
            double wavelen = 2.0 * M_PI / inv;
            double low_wl = (double)c.rope_orig_ctx / c.rope_low_freq, high_wl = (double)c.rope_orig_ctx / c.rope_high_freq;
            if (wavelen > low_wl) inv = inv / c.rope_factor;
            else if (wavelen >= high_wl) {
                double smooth = ((double)c.rope_orig_ctx / wavelen - c.rope_low_freq) / (c.rope_high_freq - c.rope_low_freq);
                inv = (1.0 - smooth) * inv / c.rope_factor + smooth * inv;
            }
        }
        for (int p = 0; p < max_pos; ++p) {
            double a = (double)p * inv;
            cosv[(size_t)p * half + i] = (float)std::cos(a); sinv[(size_t)p * half + i] = (float)std::sin(a);
        }
    }
}

// The CUDA "current device" is per host thread.  Creating or destroying an engine must not leave the CALLER's thread on another device (a
// router process owns one engine per GPU; torch / NCCL in the same process assume their own device stays current), so both restore it.
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); cudaSetDevice(dev); }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

DeviceModel::DeviceModel(const ModelConfig& c, const EngineOptions& o) : cfg(c), opt(o) {
    DeviceGuard guard(opt.device);
    cuda_check(cudaSetDevice(opt.device), "cudaSetDevice");
    cudaDeviceProp prop;
    cuda_check(cudaGetDeviceProperties(&prop, opt.device), "cudaGetDeviceProperties");
    if (prop.major != 9 || prop.minor != 0) throw std::runtime_error("opsagent_b200 requires an sm_90 (Hopper H100) device; found sm_" +
                                                   std::to_string(prop.major) + std::to_string(prop.minor));
    sm_count = prop.multiProcessorCount;
    cuda_check(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking), "cudaStreamCreate");
    tp = opt.tp; tp_rank = opt.tp_rank;
    nh_l = cfg.n_heads / tp; nkv_l = cfg.n_kv_heads / tp; F_l = cfg.ffn / tp; V_l = cfg.vocab / tp;
    const int H = cfg.hidden, L = cfg.n_layers, F = F_l, V = cfg.vocab, D = cfg.head_dim;
    const int qd = nh_l * D, kd = nkv_l * D, qkvd = qd + 2 * kd;              // this rank's shard
    const int qd_g = cfg.q_dim(), F_g = cfg.ffn;                              // logical (global) sizes for the weight generator
    const int64_t r = tp_rank;
    const float nstd = cfg.norm_random ? 0.1f : 0.0f;

    // ---- weights: seeded init directly in HBM, bit-identical to the oracle's generator ----
    embed = dmalloc((size_t)V * H * 2); weight_bytes += (size_t)V * H * 2;
    cuda_check(launch_init_weight(embed, cfg.seed, (uint64_t)L * 16 + TG_EMBED, -1, V, H, cfg.init_std, 0.f, stream), "init embed");
    final_norm = dmalloc((size_t)H * 2);
    cuda_check(launch_init_weight(final_norm, cfg.seed, (uint64_t)L * 16 + TG_NORM, -1, 1, H, nstd, 1.f, stream), "init norm");
    // LM head is vocab-parallel: this rank owns rows [r*V_l, (r+1)*V_l)
    if (cfg.tie_embeddings) { lm_head.ptr = reinterpret_cast<uint16_t*>(embed) + (size_t)r * V_l * H; lm_head.N = V_l; lm_head.K = H; make_weight_maps(lm_head); }
    else { alloc_weight(lm_head, V_l, H); cuda_check(launch_init_weight(lm_head.ptr, cfg.seed, (uint64_t)L * 16 + TG_LMHEAD, -1, V_l, H, cfg.init_std, 0.f, stream, r * V_l), "init lm_head"); }
    layers.resize(L);
    // fp8 projections: each matrix is generated (or loaded) as bf16 into one scratch the size of the largest, then quantised into its e4m3
    // allocation on the same stream; the scratch is freed once the weights are in place, so the peak stays below the bf16 engine's weights
    const bool w8 = cfg.w_fp8();
    if (w8) w8_scratch_ = dmalloc(std::max({(size_t)qkvd * H, (size_t)H * qd, (size_t)2 * F * H, (size_t)H * F}) * 2);
    for (int l = 0; l < L; ++l) {
        Layer& ly = layers[l]; const uint64_t b = (uint64_t)l * 16;
        alloc_weight(ly.qkv, qkvd, H, w8); alloc_weight(ly.o, H, qd, w8); alloc_weight(ly.gu, 2 * F, H, w8); alloc_weight(ly.down, H, F, w8);
        uint16_t* wq = bf16_dst(ly.qkv);
        // column-parallel q|k|v and gate|up (row shards), row-parallel o and down (column shards of the logical tensors)
        cuda_check(launch_init_weight(wq, cfg.seed, b + T_WQ, -1, qd, H, cfg.init_std, 0.f, stream, r * qd), "init wq");
        cuda_check(launch_init_weight(wq + (size_t)qd * H, cfg.seed, b + T_WK, -1, kd, H, cfg.init_std, 0.f, stream, r * kd), "init wk");
        cuda_check(launch_init_weight(wq + (size_t)(qd + kd) * H, cfg.seed, b + T_WV, -1, kd, H, cfg.init_std, 0.f, stream, r * kd), "init wv");
        commit(ly.qkv);
        cuda_check(launch_init_weight(bf16_dst(ly.o), cfg.seed, b + T_WO, -1, H, qd, cfg.init_std, 0.f, stream, 0, r * qd, qd_g), "init wo");
        commit(ly.o);
        cuda_check(launch_init_weight(bf16_dst(ly.gu), cfg.seed, b + T_WG, (int64_t)(b + T_WU), 2 * (int64_t)F, H, cfg.init_std, 0.f, stream, r * F), "init wgu");
        commit(ly.gu);
        cuda_check(launch_init_weight(bf16_dst(ly.down), cfg.seed, b + T_WD, -1, H, F, cfg.init_std, 0.f, stream, 0, r * F, F_g), "init wd");
        commit(ly.down);
        ly.ln1 = dmalloc((size_t)H * 2); ly.ln2 = dmalloc((size_t)H * 2);
        cuda_check(launch_init_weight(ly.ln1, cfg.seed, b + T_LN1, -1, 1, H, nstd, 1.f, stream), "init ln1");
        cuda_check(launch_init_weight(ly.ln2, cfg.seed, b + T_LN2, -1, 1, H, nstd, 1.f, stream), "init ln2");
        if (cfg.qkv_bias) {
            ly.bqkv = dmalloc((size_t)qkvd * 2);
            uint16_t* bq = reinterpret_cast<uint16_t*>(ly.bqkv);
            cuda_check(launch_init_weight(bq, cfg.seed, b + T_BQ, -1, 1, qd, cfg.init_std, 0.f, stream, 0, r * qd, qd_g), "init bq");
            cuda_check(launch_init_weight(bq + qd, cfg.seed, b + T_BK, -1, 1, kd, cfg.init_std, 0.f, stream, 0, r * kd, cfg.kv_dim()), "init bk");
            cuda_check(launch_init_weight(bq + qd + kd, cfg.seed, b + T_BV, -1, 1, kd, cfg.init_std, 0.f, stream, 0, r * kd, cfg.kv_dim()), "init bv");
        }
    }

    kv_k_scale.assign(L, 1.0f); kv_v_scale.assign(L, 1.0f);
    if (!opt.weights.empty()) load_checkpoint(opt.weights);
    if (w8_scratch_) {
        cuda_check(cudaStreamSynchronize(stream), "weight quantisation");
        cuda_check(cudaFree(w8_scratch_), "cudaFree");
        allocs_.erase(std::find(allocs_.begin(), allocs_.end(), w8_scratch_)); w8_scratch_ = nullptr;
    }

    // ---- RoPE table ----
    {
        std::vector<float> cs, sn; rope_table(cfg, opt.max_seq_len, cs, sn);
        rope_cos = reinterpret_cast<float*>(dmalloc(cs.size() * 4)); rope_sin = reinterpret_cast<float*>(dmalloc(sn.size() * 4));
        cuda_check(cudaMemcpyAsync(rope_cos, cs.data(), cs.size() * 4, cudaMemcpyHostToDevice, stream), "rope cos");
        cuda_check(cudaMemcpyAsync(rope_sin, sn.data(), sn.size() * 4, cudaMemcpyHostToDevice, stream), "rope sin");
        cuda_check(cudaStreamSynchronize(stream), "rope sync");
    }

    // ---- activations ----
    max_rows_ = std::max(opt.max_step_tokens, opt.max_batch);
    max_sample_ = std::max(opt.max_batch, std::min(max_rows_, 2048));
    const int MR = max_rows_;
    x_ = dmalloc((size_t)MR * H * 2); qkv_ = dmalloc((size_t)MR * qkvd * 2); q_ = dmalloc((size_t)MR * qd * 2);
    auto amap = [&](CUtensorMap* tm, void* p, int rows, int cols) {
        tmap_check(make_tmap_bf16_2d(tm, p, (uint64_t)rows, (uint64_t)cols, (uint64_t)cols, 128, 64), "an activation buffer");
    };
    // projection inputs, zeroed (as their e4m3 copies): the GEMMs' stale rows stay finite
    for (const auto& [a, cols] : {std::make_pair(&xn_, H), std::make_pair(&attn_, qd), std::make_pair(&act_, F)}) {
        a->cols = cols;
        a->x = dmalloc((size_t)MR * cols * 2);
        cuda_check(cudaMemsetAsync(a->x, 0, (size_t)MR * cols * 2, stream), "memset");
        amap(&a->tm, a->x, MR, cols);
        if (!w8) continue;
        a->q = reinterpret_cast<uint8_t*>(dmalloc((size_t)MR * cols)); a->sc = reinterpret_cast<float*>(dmalloc((size_t)MR * 4));
        cuda_check(cudaMemsetAsync(a->q, 0, (size_t)MR * cols, stream), "memset"); cuda_check(cudaMemsetAsync(a->sc, 0, (size_t)MR * 4, stream), "memset");
        tmap_check(make_tmap_u8_2d(&a->tm8, a->q, (uint64_t)MR, (uint64_t)cols, 128, 128), "an fp8 activation buffer");
    }
    cuda_check(cudaMemsetAsync(q_, 0, (size_t)MR * qd * 2, stream), "memset");
    // sampled rows (debug logits sample every row of a short prefill: up to 2048)
    const int MS = max_sample_;
    xs_ = dmalloc((size_t)MS * H * 2); xsn_ = dmalloc((size_t)MS * H * 2);
    cuda_check(cudaMemsetAsync(xsn_, 0, (size_t)MS * H * 2, stream), "memset");
    amap(&tm_xsn_, xsn_, MS, H);
    const int lm_tiles_max = gemm_n_tiles(V_l, 32);
    amax_val_ = reinterpret_cast<float*>(dmalloc((size_t)MS * lm_tiles_max * 4));
    amax_idx_ = reinterpret_cast<int*>(dmalloc((size_t)MS * lm_tiles_max * 4));
    d_out_ids_ = reinterpret_cast<int32_t*>(dmalloc((size_t)MS * 4));
    // token-mask table of the grammar-constrained decoder: one bitset over the whole vocabulary per cached automaton state
    mask_words = (cfg.vocab + 31) / 32;
    mask_slots = std::max(1024, 2 * opt.max_batch);
    max_mask_updates = opt.max_batch;               // a scheduler step samples at most one row per running sequence
    mask_table_ = reinterpret_cast<uint32_t*>(dmalloc((size_t)mask_slots * mask_words * 4));
    cuda_check(cudaMemsetAsync(mask_table_, 0, (size_t)mask_slots * mask_words * 4, stream), "mask table memset");
    cuda_check(cudaMallocHost(&h_out_ids, (size_t)MS * 4), "cudaMallocHost");

    // ---- paged KV pool ----
    const size_t page_bytes = (size_t)2 * L * nkv_l * 64 * D * cfg.kv_elem_bytes();    // all layers, K and V, of 64 tokens (this rank's kv heads)
    if (opt.num_pages > 0) num_pages = opt.num_pages;
    else {
        size_t free_b = 0, total_b = 0;
        cuda_check(cudaMemGetInfo(&free_b, &total_b), "cudaMemGetInfo");
        double budget = opt.kv_gb > 0 ? opt.kv_gb * 1e9 : (double)free_b - 6e9;
        budget = std::min(budget, (double)free_b - 2e9);
        num_pages = (int)std::max(0.0, budget / (double)page_bytes);
    }
    max_pages_per_seq = opt.max_seq_len / 64;
    if (num_pages < max_pages_per_seq) throw std::runtime_error("KV pool too small: " + std::to_string(num_pages) + " pages < one max-length sequence");
    const int64_t plane_rows = (int64_t)num_pages * nkv_l * 64;
    if ((double)plane_rows * 2 * L >= 2147483647.0) { num_pages = (int)(2147483647.0 / (2.0 * L * nkv_l * 64)) - 1; }
    kv.page_size = 64; kv.n_kv = nkv_l; kv.head_dim = D; kv.num_pages = num_pages;
    kv.kv_stride_rows = (int64_t)num_pages * nkv_l * 64; kv.layer_stride_rows = 2 * kv.kv_stride_rows;
    kv.fp8 = cfg.kv_fp8(); kv.k_scale = kv_k_scale.data(); kv.v_scale = kv_v_scale.data();
    kv_pool_bytes = (size_t)num_pages * page_bytes;
    kv.base = dmalloc(kv_pool_bytes);
    cuda_check(cudaMemsetAsync(kv.base, 0, kv_pool_bytes, stream), "kv memset");   // stale pages must hold finite values (0*NaN; e4m3 0x00 = +0)
    {
        // fp8: the pool as rows of 128 bytes, one (page, kv head) block of K or V per box
        tmap_check(kv.fp8 ? make_tmap_u8_2d(&tm_kv, kv.base, (uint64_t)(kv_pool_bytes / 128), 128, (uint32_t)(D / 2), 128)
                          : make_tmap_bf16_2d(&tm_kv, kv.base, (uint64_t)kv.layer_stride_rows * L, (uint64_t)D, (uint64_t)D, 64, 64), "the KV pool");
    }

    // ---- decode-attention partial workspace + per-step metadata arena ----
    const int n_ctas = opt.attn_ctas > 0 ? opt.attn_ctas : 2 * sm_count;
    max_part_slots_ = 2 * n_ctas + 2 * opt.max_batch * nkv_l + 16;
    const int grp = cfg.n_heads / cfg.n_kv_heads;
    part_o_ = reinterpret_cast<float*>(dmalloc((size_t)max_part_slots_ * grp * D * 4));
    part_ml_ = reinterpret_cast<float*>(dmalloc((size_t)max_part_slots_ * grp * 2 * 4));
    meta_cap_words_ = (size_t)4 * MR + (size_t)opt.max_batch * (max_pages_per_seq + 2) + (size_t)MR / 64 * 4 + 4 * opt.max_batch +
                      (size_t)(opt.max_batch * nkv_l + n_ctas + 8) * 8 * 2 + (size_t)n_ctas + 4096 + (size_t)max_sample_ + (size_t)max_mask_updates * (mask_words + 4);
    for (int i = 0; i < 2; ++i) {
        cuda_check(cudaMallocHost(&h_meta_buf_[i], meta_cap_words_ * 4), "cudaMallocHost meta");
        cuda_check(cudaEventCreateWithFlags(&meta_ev_[i], cudaEventDisableTiming), "cudaEventCreate meta");
    }
    h_meta_ = h_meta_buf_[0];
    d_meta_ = reinterpret_cast<int32_t*>(dmalloc(meta_cap_words_ * 4));
    sk_bn_ = (opt.sk_bn == 256) ? 256 : 128;
    sk_G_ = opt.sk_ctas > 0 ? opt.sk_ctas : sm_count;
    {
        size_t wsb = 0;
        for (int n : {qkvd, H, 2 * F}) { wsb = std::max(wsb, streamk_ws_bytes(n, 256, sk_G_, 128)); wsb = std::max(wsb, streamk_ws_bytes(n, 128, sk_G_, 256)); wsb = std::max(wsb, streamk_ws_bytes(n, 64, sk_G_, 128)); }
        sk_ws_ = reinterpret_cast<float*>(dmalloc(wsb));
        tile_flags_ = reinterpret_cast<unsigned int*>(dmalloc((size_t)4 * SK_MAX_FLAG_TILES * 4));
        cuda_check(cudaMemset(tile_flags_, 0, (size_t)4 * SK_MAX_FLAG_TILES * 4), "stream-K tile flags memset");
        // 32-bit index arithmetic in the consumers: (units of the largest shape + kb) * G must stay below 2^32
        const double worst = ((double)((2 * F + sk_bn_ - 1) / sk_bn_) * ((std::max(H, F) + 63) / 64) + (std::max(H, F) + 63) / 64) * sk_G_;
        if (worst >= 4.0e9) throw std::runtime_error("stream-K index range exceeds 32 bits for this model");
    }
    ev.resize(2 * (size_t)L);
    for (auto& e : ev) cuda_check(cudaEventCreate(&e), "cudaEventCreate");
    if (tp > 1) {
        if (opt.num_pages <= 0) throw std::runtime_error("tensor parallel engines need an explicit num_pages (all ranks must agree on the pool size)");
        // bf16 prefill partials | fp32 decode partials | up to 256 rows of this rank's fp32 logits shard (debug parity hook)
        const size_t sym_bytes = std::max({(size_t)MR * H * 2, (size_t)256 * H * 4, (size_t)256 * V_l * 4});
        // NVLS buffer: two partial + two reduced regions of 128 rows x H fp32 (decode batches: <= 128 rows on the stream-K path)
        nvls_region_ = (size_t)128 * H * 4;
        comm.reset(new TpComm(tp, tp_rank, opt.tp_shm, sym_bytes, max_sample_, opt.tp_nonce, opt.tp_nvls ? 4 * nvls_region_ + 4096 : 0));      // + per-row flags: [2 buffers][128 rows] uint32 epochs
    }
    cuda_check(cudaStreamSynchronize(stream), "init sync");
}

// ---- Hugging Face checkpoint loading (checkpoint.hpp assembles this rank's rows on the host) -------------------------------------------
void DeviceModel::load_checkpoint(const std::string& path) {
    SafeTensors st(path);
    const bool w8 = cfg.w_fp8();
    if (cfg.kv_fp8()) load_kv_scales(st, cfg.n_layers, kv_k_scale, kv_v_scale);
    const CkptShard shard(st, cfg, tp, tp_rank);
    std::vector<uint16_t> hb; std::vector<uint8_t> hq; std::vector<float> hs;
    // every copy runs on `stream`, after the seeded init it overwrites, and lands before its host buffer is refilled: a pageable cudaMemcpy
    // may return before its DMA lands, and it does not order with a non-blocking stream
    auto h2d = [&](void* dst, const void* src, size_t bytes) { cuda_check(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream), "checkpoint H2D"); };
    auto landed = [&]() { cuda_check(cudaStreamSynchronize(stream), "checkpoint H2D"); };
    auto load = [&](const CkptRows& m, void* dst) { ckpt_bf16(st, m, hb); h2d(dst, hb.data(), hb.size() * 2); landed(); };
    // a projection: bf16 / F16 / F32 parts through the same bf16 destination + commit as the seeded init; F8_E4M3 parts bring bytes and scales
    auto load_proj = [&](WeightMat& w, const CkptRows& m) {
        if (!ckpt_is_f8(st, m, w8)) { load(m, bf16_dst(w)); commit(w); return; }
        ckpt_f8(st, m, hq, hs); h2d(w.ptr, hq.data(), hq.size()); h2d(w.sw, hs.data(), hs.size() * 4); landed();
    };
    load(shard.embed, embed);
    load(shard.norm, final_norm);
    if (!cfg.tie_embeddings) load(shard.lm_head, lm_head.ptr);
    for (int l = 0; l < cfg.n_layers; ++l) {
        Layer& ly = layers[l]; const CkptLayerRows& m = shard.layers[l];
        load_proj(ly.qkv, m.qkv); load_proj(ly.o, m.o); load_proj(ly.gu, m.gu); load_proj(ly.down, m.down);
        load(m.ln1, ly.ln1); load(m.ln2, ly.ln2);
        if (cfg.qkv_bias) load(m.bqkv, ly.bqkv);
    }
}

DeviceModel::~DeviceModel() {
    DeviceGuard guard(opt.device);
    if (stream) cudaStreamSynchronize(stream);
    for (auto& e : ev) cudaEventDestroy(e);
    for (void* p : allocs_) cudaFree(p);
    if (h_out_ids) cudaFreeHost(h_out_ids);
    for (int i = 0; i < 2; ++i) { if (h_meta_buf_[i]) cudaFreeHost(h_meta_buf_[i]); if (meta_ev_[i]) cudaEventDestroy(meta_ev_[i]); }
    comm.reset();                 // peer mappings and symmetric buffers: released while this engine's device is still current
    if (stream) cudaStreamDestroy(stream);
}

const char* DeviceModel::kt_name(int id) {
    static const char* n[16] = {"h2d+embed", "rmsnorm", "qkv_gemm", "rope_kv", "attention", "attn_merge", "o_gemm", "resid_rmsnorm", "gate_up_gemm",
                                "swiglu", "down_gemm", "gather+norm", "lm_head", "argmax+d2h", "fp8_quant", ""};
    return n[id & 15];
}
void DeviceModel::sync() { cuda_check(cudaStreamSynchronize(stream), "stream sync"); }
void DeviceModel::sampled_logits(int S, float* out) {
    const int n_tiles = gemm_n_tiles(cfg.vocab, pick_bn(S, cfg.vocab, sm_count, opt.bn_lm));     // the LM head's per-tile row maxima of that forward
    std::vector<float> v((size_t)S * n_tiles);
    cuda_check(cudaMemcpy(v.data(), amax_val_, v.size() * 4, cudaMemcpyDeviceToHost), "row maxima D2H");
    for (int r = 0; r < S; ++r) out[r] = *std::max_element(v.begin() + (size_t)r * n_tiles, v.begin() + (size_t)(r + 1) * n_tiles);
}

// N-tile heuristic.  Decode (M <= 128) streams weights once: prefer the largest tile that still yields >= 1 CTA
// per SM; prefill has M/128 row tiles as well, so the widest tile (least A re-reads) wins.
int pick_bn(int M, int N, int sm_count, int override_bn, bool fp8) {
    if (fp8) return std::min(pick_bn(M, N, sm_count, override_bn), W8_MAX_BN);
    if (override_bn == 32 || override_bn == 64 || override_bn == 128 || override_bn == 256) return override_bn;
    const int m_tiles = (M + 127) / 128;
    // no 256-wide tile: its 64 x 256 fp32 fragment does not fit one consumer warpgroup's registers without spills
    const int cands[3] = {128, 64, 32};
    // one or two row tiles (decode-sized batches off the stream-K path, e.g. Qwen2.5-32B TP=4 at B=256): a CTA's k-loop is latency-bound,
    // so wider tiles with fewer, longer-lived CTAs win as long as about half the SMs stream; many row tiles: fill every SM
    const long long want = m_tiles <= 2 ? sm_count / 2 : sm_count;
    for (int bn : cands) { if ((long long)((N + bn - 1) / bn) * m_tiles >= want) return bn; }
    return 32;
}

void append_prefill_tiles(std::vector<PrefillTile>& tiles, int seq, int row0, int pos0, int n_rows) {
    for (int r = 0; r < n_rows; r += PREFILL_TILE_ROWS) tiles.push_back(PrefillTile{seq, row0 + r, pos0 + r, std::min(PREFILL_TILE_ROWS, n_rows - r)});
}

void sort_prefill_tiles(std::vector<PrefillTile>& tiles) {
    // the causal triangle otherwise leaves a long tail of big CTAs
    std::stable_sort(tiles.begin(), tiles.end(), [](const PrefillTile& a, const PrefillTile& b) { return a.pos0 + a.n_rows > b.pos0 + b.n_rows; });
}

void build_decode_plan(const int32_t* ctx_lens, int n_seqs, int n_kv, int n_ctas_target, int force_splits, DecodePlan& out) {
    out.segs.clear(); out.cta_ptr.clear(); out.merges.clear(); out.n_slots = 0;
    long long total = 0;
    for (int i = 0; i < n_seqs; ++i) total += (long long)((ctx_lens[i] + 63) / 64) * n_kv;
    if (total <= 0) { out.cta_ptr.push_back(0); return; }
    if (force_splits > 0) {
        // test mode: every (seq, kvh) item is cut into `force_splits` pieces, one CTA per piece
        out.cta_ptr.push_back(0);
        for (int s = 0; s < n_seqs; ++s) for (int h = 0; h < n_kv; ++h) {
            const int nch = (ctx_lens[s] + 63) / 64; if (nch == 0) continue;
            const int pieces = std::min(force_splits, nch), per = (nch + pieces - 1) / pieces;
            const int real = (nch + per - 1) / per;
            MergeItem mi{s, h, out.n_slots, real};
            const int slot0 = out.n_slots, item = (int)out.merges.size();
            for (int pz = 0; pz < real; ++pz) {
                DecodeSeg sg{s, h, pz * per, std::min(nch, (pz + 1) * per), real > 1 ? out.n_slots++ : -1, slot0, real, item};
                out.segs.push_back(sg); out.cta_ptr.push_back((int32_t)out.segs.size());
            }
            if (real > 1) out.merges.push_back(mi);
        }
        return;
    }
    long long n_ctas = std::min<long long>(n_ctas_target, std::max<long long>(1, total / 2));
    const long long per = (total + n_ctas - 1) / n_ctas;
    n_ctas = (total + per - 1) / per;
    out.cta_ptr.assign((size_t)n_ctas + 1, 0);
    long long gpos = 0;   // global chunk cursor
    std::vector<int> cta_of_seg;
    for (int s = 0; s < n_seqs; ++s) for (int h = 0; h < n_kv; ++h) {
        const int nch = (ctx_lens[s] + 63) / 64; if (nch == 0) continue;
        const long long g0 = gpos, g1 = gpos + nch;
        const long long c_first = g0 / per, c_last = (g1 - 1) / per;
        const int pieces = (int)(c_last - c_first + 1);
        MergeItem mi{s, h, out.n_slots, pieces};
        const int slot0 = out.n_slots, item = (int)out.merges.size();
        for (long long c = c_first; c <= c_last; ++c) {
            const long long a = std::max(g0, c * per), b = std::min(g1, (c + 1) * per);
            DecodeSeg sg{s, h, (int32_t)(a - g0), (int32_t)(b - g0), pieces > 1 ? out.n_slots++ : -1, slot0, pieces, item};
            out.segs.push_back(sg); cta_of_seg.push_back((int)c);
        }
        if (pieces > 1) out.merges.push_back(mi);
        gpos = g1;
    }
    // segs are already ordered by CTA; build the CSR pointer
    size_t k = 0;
    for (long long c = 0; c < n_ctas; ++c) {
        out.cta_ptr[(size_t)c] = (int32_t)k;
        while (k < cta_of_seg.size() && cta_of_seg[k] == c) ++k;
    }
    out.cta_ptr[(size_t)n_ctas] = (int32_t)k;
}

void DeviceModel::forward(const StepInput& in, float* logits_out) {
    const int T = (int)in.tokens.size(), S = (int)in.sample_rows.size();
    // all projection sizes below are this rank's shard (== the global sizes when tp == 1)
    const int H = cfg.hidden, L = cfg.n_layers, F = F_l, V = V_l, D = cfg.head_dim;
    const int nh = nh_l, nkv = nkv_l, qd = nh * D, qkvd = qd + 2 * nkv * D;
    const bool use_tp = tp > 1;
    if (T <= 0 || T > max_rows_ || S > max_sample_) throw std::runtime_error("forward: bad batch size");
    if (in.decode && in.n_seqs != T) throw std::runtime_error("forward: decode needs one token per sequence");

    // ---- pack per-step metadata into one pinned arena, one H2D copy ----
    meta_idx_ ^= 1; h_meta_ = h_meta_buf_[meta_idx_];
    cuda_check(cudaEventSynchronize(meta_ev_[meta_idx_]), "meta staging fence");     // its previous H2D copy has been consumed
    size_t w = 0;
    auto put = [&](const void* src, size_t words) -> size_t {
        size_t at = w; if (at + words > meta_cap_words_) throw std::runtime_error("forward: metadata arena overflow");
        if (words) std::memcpy(h_meta_ + at, src, words * 4);
        w = (at + words + 3) & ~size_t(3); return at;
    };
    const size_t o_tok = put(in.tokens.data(), T), o_pos = put(in.positions.data(), T), o_slot = put(in.slots.data(), T);
    const size_t o_samp = put(in.sample_rows.data(), S);
    const size_t o_bt = put(in.block_tables.data(), in.block_tables.size());
    const size_t o_ctx = put(in.ctx_lens.data(), in.ctx_lens.size());
    if (!in.mask_slots.empty() && (int)in.mask_slots.size() != S) throw std::runtime_error("forward: mask_slots must be [n_sample]");
    const size_t rec = (size_t)mask_words + 1, n_upd = in.mask_updates.size() / rec;
    if (in.mask_updates.size() % rec != 0 || (int)n_upd > max_mask_updates) throw std::runtime_error("forward: malformed or too many token-mask updates");
    for (int ms : in.mask_slots) if (ms >= mask_slots) throw std::runtime_error("forward: token-mask slot out of range");
    const size_t o_mslot = put(in.mask_slots.data(), in.mask_slots.size());
    const size_t o_mupd = put(in.mask_updates.data(), in.mask_updates.size());
    size_t o_segs = 0, o_ptr = 0, o_tiles = 0, o_cnt = 0;
    const int n_dec = in.decode ? in.n_seqs : in.n_decode;          // sequences served by the decode attention kernel (rows 0..n_dec-1)
    if (n_dec < 0 || n_dec > in.n_seqs || n_dec > T) throw std::runtime_error("forward: bad n_decode");
    if (n_dec > 0) {
        const int n_ctas = opt.attn_ctas > 0 ? opt.attn_ctas : 2 * sm_count;
        build_decode_plan(in.ctx_lens.data(), n_dec, nkv, n_ctas, 0, plan_);
        if (plan_.n_slots > max_part_slots_) throw std::runtime_error("forward: partial workspace overflow");
        o_segs = put(plan_.segs.data(), plan_.segs.size() * 8);
        o_ptr = put(plan_.cta_ptr.data(), plan_.cta_ptr.size());
        zero_counters_.assign(plan_.merges.size() + 1, 0);
        o_cnt = put(zero_counters_.data(), zero_counters_.size());     // merge counters start every step at zero
    }
    if (!in.decode) {
        sorted_tiles_ = in.tiles;
        sort_prefill_tiles(sorted_tiles_);
        o_tiles = put(sorted_tiles_.data(), sorted_tiles_.size() * 4);
    }
    cuda_check(cudaMemcpyAsync(d_meta_, h_meta_, w * 4, cudaMemcpyHostToDevice, stream), "meta H2D");
    for (size_t u = 0; u < n_upd; ++u) {           // new automaton states: bitset rows of the device table (read by the LM-head epilogue below)
        const uint32_t slot = in.mask_updates[u * rec];
        if ((int)slot >= mask_slots) throw std::runtime_error("forward: token-mask update slot out of range");
        cuda_check(cudaMemcpyAsync(mask_table_ + (size_t)slot * mask_words, d_meta_ + o_mupd + u * rec + 1, (size_t)mask_words * 4, cudaMemcpyDeviceToDevice, stream), "token-mask update");
    }
    cuda_check(cudaEventRecord(meta_ev_[meta_idx_], stream), "meta event");
    h2d_bytes += w * 4;
    const int32_t* d_tok = d_meta_ + o_tok; const int32_t* d_pos = d_meta_ + o_pos; const int32_t* d_slot = d_meta_ + o_slot;
    const int32_t* d_samp = d_meta_ + o_samp; const int32_t* d_bt = d_meta_ + o_bt; const int32_t* d_ctx = d_meta_ + o_ctx;

    size_t ek = 0;
    if (profile_all) {
        const size_t n_ev = (size_t)L * (cfg.w_fp8() ? 16 : 12) + 16;      // fp8: four quantiser launches per layer
        if (ev_all.size() < n_ev) { size_t o = ev_all.size(); ev_all.resize(n_ev); for (size_t i = o; i < ev_all.size(); ++i) cudaEventCreate(&ev_all[i]); }
        ev_ids.assign(ev_all.size(), 0);
        cudaEventRecord(ev_all[ek++], stream);
    }
    auto MARK = [&](int id) { if (profile_all && ek < ev_all.size()) { ev_ids[ek] = id; cudaEventRecord(ev_all[ek++], stream); } };
    const Mark mark = profile_all ? Mark(MARK) : Mark();       // the stage functions' marks
    cuda_check(launch_embed_gather(d_tok, embed, x_, T, H, cfg.vocab, stream), "embed"); MARK(0);
    // fp8 weights: every projection reads its input as e4m3 rows + per-row scales, quantised by one kernel right before the GEMM
    const bool w8 = cfg.w_fp8();
    auto quant = [&](const ProjInput& a) { if (a.q) { cuda_check(launch_quant_rows_e4m3(a.x, a.q, a.sc, T, a.cols, stream), "fp8 quantise"); MARK(14); } };
    auto cap = [&](int bn) { return w8 ? std::min(bn, W8_MAX_BN) : bn; };
    // decode-sized batches (one or, opt-in, two 128-row tiles; fp8: one, the promoted fp8 fragment leaves no registers for a second)
    const bool use_sk = opt.streamk && T <= (w8 ? 128 : std::min(256, std::max(128, opt.sk_max_rows)));
    const int sk_rows = T > 128 ? 256 : 128;
    // rows 0 .. n_dec-1: decode attention, cut items merged inside the kernel by the CTA finishing their last piece; then the prefill tiles
    const DecodeAttnParams dec{q_, attn_.x, d_bt, d_ctx, max_pages_per_seq, reinterpret_cast<const DecodeSeg*>(d_meta_ + o_segs), d_meta_ + o_ptr,
                               n_dec > 0 ? (int)plan_.cta_ptr.size() - 1 : 0, part_o_, part_ml_, d_meta_ + o_cnt, 0, nh, nkv, 0.f};
    const PrefillAttnParams pre{q_, attn_.x, d_bt, max_pages_per_seq, reinterpret_cast<const PrefillTile*>(d_meta_ + o_tiles),
                                in.decode ? 0 : (int)in.tiles.size(), 0, nh, nkv, 0.f};
    auto attention = [&](int l) {
        if (profile_attn) cudaEventRecord(ev[2 * l], stream);
        step_attention(&tm_kv, kv, dec, pre, l, stream, mark);
        if (profile_attn) cudaEventRecord(ev[2 * l + 1], stream);
    };
    if (use_sk) {
        // decode-sized batch: persistent stream-K projections (fp32 partials) + fused consumers
        auto bn_of = [&](int o) { return cap(sk_rows == 256 ? 128 : ((o == 64 || o == 128 || o == 256) ? o : sk_bn_)); };      // two row tiles need BN <= 128 (registers)
        auto sk_for = [&](int N, int K, int o) {        // the GEMM prefetches its first weight tiles into L2
            StreamK k = make_streamk(sk_ws_, N, K, bn_of(o), sk_G_, sk_rows, w8); k.l2_prefetch_units = std::max(0, opt.sk_l2_prefetch_kb * 1024 / (k.bn * 128)); return k;
        };
        const StreamK sk_qkv = sk_for(qkvd, H, opt.sk_bn_qkv), sk_o = sk_for(H, qd, opt.sk_bn_o), sk_gu = sk_for(2 * F, H, opt.sk_bn_gu), sk_dn = sk_for(H, F, opt.sk_bn_down);
        cuda_check(launch_rmsnorm(x_, layers[0].ln1, xn_.x, T, H, cfg.rms_eps, stream), "rmsnorm1"); MARK(1);
        // qkv / o / down epilogues finished inside the GEMM (same conditions as the fused SwiGLU; every projection at BN = 128, tile counts within the flag arrays)
        const bool fuse_ok = sk_rows == 128 && sk_G_ <= sm_count && sk_qkv.bn == 128 && sk_o.bn == 128 && sk_dn.bn == 128 &&
                              sk_qkv.n_tiles <= SK_MAX_FLAG_TILES && sk_o.n_tiles <= SK_MAX_FLAG_TILES && (D == 64 || D == 128);
        const bool fuse_rope = fuse_ok && (opt.sk_fuse_epi & 1), fuse_o = fuse_ok && !use_tp && (opt.sk_fuse_epi & 2), fuse_dn = fuse_ok && !use_tp && (opt.sk_fuse_epi & 4);
        // cluster split-K (few-tile projections): cluster size per shape, 0 = keep stream-K.  o / down finish the residual add themselves, so
        // they are single-GPU only (a tensor-parallel rank must hand its partial to the all-reduce instead)
        const int ck_qkv = (sk_rows == 128 && (opt.sk_clusterk & 1) && (D == 64 || D == 128)) ? clusterk_pick(qkvd, H, sm_count, opt.sk_clusterk_min_fill) : 0;
        const int ck_o = (sk_rows == 128 && (opt.sk_clusterk & 2) && !use_tp) ? clusterk_pick(H, qd, sm_count, opt.sk_clusterk_min_fill) : 0;
        const int ck_dn = (sk_rows == 128 && (opt.sk_clusterk & 4) && !use_tp) ? clusterk_pick(H, F, sm_count, opt.sk_clusterk_min_fill) : 0;
        const bool fuse_swiglu = opt.sk_fuse_swiglu && !w8 && sk_rows == 128 && sk_gu.bn == 128 && sk_G_ <= sm_count && sk_gu.n_tiles <= SK_MAX_FLAG_TILES;
        // each projection's finishing path (stages.hpp): cluster split-K, fused stream-K finisher, or GEMM + consumer
        const int path_qkv = ck_qkv ? ck_qkv : fuse_rope, path_o = ck_o ? ck_o : fuse_o, path_dn = ck_dn ? ck_dn : fuse_dn, path_gu = fuse_swiglu;
        auto proj = [&](int path, const ProjInput& a, const WeightMat& w, const StreamK& sk, int flag_slot) {
            return SkGemm{path, a.map(), w.map(path == 0 ? sk.bn : 128), T, w.N, w.K, sk, a.w8(w), tile_flags_ + flag_slot * SK_MAX_FLAG_TILES};
        };
        // row-parallel projection (o, down): x += a . w^T, then xn = rmsnorm(x) * gain
        auto row_parallel = [&](const ProjInput& a, const WeightMat& w, int path, const StreamK& sk, int flag_slot, const void* gain, const RowParallelOp& op) {
            const SkGemm g = proj(path, a, w, sk, flag_slot);
            if (!use_tp) return finish_row_parallel(g, x_, gain, xn_.x, cfg.rms_eps, op, stream, mark);
            // all-reduce the rank partials over NVLink peer memory, then residual + norm
            const int b = comm->next_buffer();
            const TpComm::Signal sg = comm->next_signal();     // "buffer written" handshake rides on the two kernels: no barrier launch
            if (comm->nvls() && T <= 128) {
                char* loc = reinterpret_cast<char*>(comm->nvls_local());
                cuda_check(launch_gemm_streamk(g.tmA, g.tmB, T, H, g.K, sk, stream, g.w8), op.gemm); MARK(op.mark);
                cuda_check(launch_sk_reduce_f32(sk, reinterpret_cast<float*>(loc + (size_t)b * nvls_region_), T, H, stream, &sg), op.nvls_part);
                cuda_check(launch_ar_nvls_resid_rmsnorm(comm->nvls_multicast(), loc, (size_t)b * nvls_region_, (size_t)(2 + b) * nvls_region_, 4 * nvls_region_ + (size_t)b * 512, tp, tp_rank,
                                                        x_, gain, xn_.x, T, H, cfg.rms_eps, stream, sg), op.nvls_ar);
                MARK(7);
                return;
            }
            tp_row_parallel_partial(g, opt.tp_ar_bf16, comm->sym(b), sg, op, stream, mark);
            tp_row_parallel_finish(comm->d_peer_sym(b), tp, opt.tp_ar_bf16, x_, gain, xn_.x, T, H, cfg.rms_eps, sg, op, stream, mark);
        };
        for (int l = 0; l < L; ++l) {
            const Layer& ly = layers[l];
            quant(xn_);
            qkv_rope(proj(path_qkv, xn_, ly.qkv, sk_qkv, 0), ly.bqkv, d_pos, d_slot, rope_cos, rope_sin, q_, kv, l, nh, stream, mark);
            attention(l);
            quant(attn_);
            row_parallel(attn_, ly.o, path_o, sk_o, 1, ly.ln2, kOProj);
            quant(xn_);
            gate_up_swiglu(proj(path_gu, xn_, ly.gu, sk_gu, 2), act_.x, stream, mark);
            quant(act_);
            row_parallel(act_, ly.down, path_dn, sk_dn, 3, (l + 1 < L) ? layers[l + 1].ln1 : final_norm, kDownProj);
        }
    } else {
        // row-parallel projection (o, down) into x.  Single GPU: the residual add in the epilogue.  Tensor parallel: bf16 partial -> symmetric
        // buffer, barrier, x += sum over ranks (rank order)
        auto row_parallel = [&](const ProjInput& a, const WeightMat& w, int K, int bn, int mark_id, const char* label) {
            if (!use_tp) {
                proj_gemm(a.map(), w.map(bn), T, H, K, EPI_RESID, bn, x_, nullptr, x_, a.w8(w), label, stream); MARK(mark_id);
                return;
            }
            const int b = comm->next_buffer();
            proj_gemm(a.map(), w.map(bn), T, H, K, EPI_STORE, bn, comm->sym(b), nullptr, nullptr, a.w8(w), label, stream); MARK(mark_id);
            cuda_check(comm->barrier(stream), "xgpu barrier");
            if (T >= opt.tp_two_shot_rows) {
                cuda_check(launch_ar2_reduce_scatter(comm->d_peer_sym(b), tp, tp_rank, x_, comm->sym(TpComm::GATHER), T, H, stream), "reduce-scatter+resid");
                cuda_check(comm->barrier(stream), "xgpu barrier");
                cuda_check(launch_ar2_all_gather(comm->d_peer_sym(TpComm::GATHER), tp, tp_rank, x_, T, H, stream), "all-gather");
            } else {
                cuda_check(launch_ar_resid_bf16(comm->d_peer_sym(b), tp, x_, T, H, stream), "allreduce+resid");
            }
        };
        const int bn_qkv = pick_bn(T, qkvd, sm_count, opt.bn_qkv, w8), bn_o = pick_bn(T, H, sm_count, opt.bn_o, w8);
        const int bn_gu = pick_bn(T, 2 * F, sm_count, opt.bn_gu, w8), bn_down = pick_bn(T, H, sm_count, opt.bn_down, w8);
        for (int l = 0; l < L; ++l) {
            const Layer& ly = layers[l];
            cuda_check(launch_rmsnorm(x_, ly.ln1, xn_.x, T, H, cfg.rms_eps, stream), "rmsnorm1"); MARK(1);
            quant(xn_);
            proj_gemm(xn_.map(), ly.qkv.map(bn_qkv), T, qkvd, H, EPI_STORE, bn_qkv, qkv_, ly.bqkv, nullptr, xn_.w8(ly.qkv), "qkv gemm", stream); MARK(2);
            cuda_check(launch_rope_kv_write(qkv_, d_pos, d_slot, rope_cos, rope_sin, q_, kv, l, T, nh, stream), "rope"); MARK(3);
            attention(l);
            quant(attn_);
            row_parallel(attn_, ly.o, qd, bn_o, 6, "o gemm");
            cuda_check(launch_rmsnorm(x_, ly.ln2, xn_.x, T, H, cfg.rms_eps, stream), "rmsnorm2"); MARK(1);
            quant(xn_);
            proj_gemm(xn_.map(), ly.gu.map(bn_gu), T, 2 * F, H, EPI_SWIGLU, bn_gu, act_.x, nullptr, nullptr, xn_.w8(ly.gu), "gate_up gemm", stream); MARK(8);
            quant(act_);
            row_parallel(act_, ly.down, F, bn_down, 10, "down gemm");
        }
    }
    if (S > 0) {
        if (use_sk) {      // xn_ already holds final_norm(x): just pick the sampled rows
            cuda_check(launch_gather_rows(xn_.x, d_samp, xsn_, S, H, stream), "gather");
        } else {
            cuda_check(launch_gather_rows(x_, d_samp, xs_, S, H, stream), "gather");
            cuda_check(launch_rmsnorm(xs_, final_norm, xsn_, S, H, cfg.rms_eps, stream), "final norm");
        }
        MARK(11);
        const int bn_lm = pick_bn(S, V, sm_count, opt.bn_lm);
        // constrained rows: the arg-max runs over their state's allowed tokens, on every vocabulary shard
        const bool masked = !in.mask_slots.empty();
        float* logits = logits_out;
        int lb = -1;
        if (use_tp) {          // vocab-parallel head: each rank's fp32 logits shard is staged in its symmetric buffer when asked for
            logits = nullptr;
            if (in.want_logits) {
                if ((size_t)S * V * 4 > comm->sym_bytes()) throw std::runtime_error("debug logits do not fit the symmetric buffer");
                lb = comm->next_buffer(); logits = reinterpret_cast<float*>(comm->sym(lb));
            }
        }
        const int b = use_tp ? comm->next_buffer() : 0;
        lm_head_argmax(&tm_xsn_, lm_head.map(bn_lm), S, V, H, bn_lm, logits, V, amax_val_, amax_idx_, masked ? mask_table_ : nullptr,
                       masked ? d_meta_ + o_mslot : nullptr, masked ? mask_words : 0, tp_rank * V, d_out_ids_, use_tp ? comm->arg(b) : nullptr, stream, mark);
        if (use_tp) {
            cuda_check(comm->barrier(stream), "xgpu barrier");
            cuda_check(launch_ar_argmax(comm->d_peer_arg(b), tp, S, d_out_ids_, stream), "argmax (all ranks)");
            if (lb >= 0 && logits_out) {   // leader assembles the full [S, vocab] logits from the peers' shards over NVLink
                for (int p = 0; p < tp; ++p)
                    cuda_check(cudaMemcpy2DAsync(logits_out + (size_t)p * V, (size_t)cfg.vocab * 4, comm->peer_sym_host(lb, p), (size_t)V * 4, (size_t)V * 4, S,
                                                 cudaMemcpyDeviceToDevice, stream), "logits gather");
            }
            if (lb >= 0) cuda_check(comm->barrier(stream), "xgpu barrier");     // peers must not reuse the staged shard before the leader has read it
        }
        cuda_check(cudaMemcpyAsync(h_out_ids, d_out_ids_, (size_t)S * 4, cudaMemcpyDeviceToHost, stream), "ids D2H"); MARK(13);
        d2h_bytes += (size_t)S * 4;
    }
    if (profile_all) {
        cuda_check(cudaStreamSynchronize(stream), "profile sync");
        for (size_t i = 1; i < ek; ++i) { float ms = 0; cudaEventElapsedTime(&ms, ev_all[i - 1], ev_all[i]); kt_ms[ev_ids[i] & 15] += ms; kt_n[ev_ids[i] & 15]++; }
    }
    if (profile_attn) {
        cuda_check(cudaStreamSynchronize(stream), "profile sync");
        for (int l = 0; l < L; ++l) { float ms = 0; cudaEventElapsedTime(&ms, ev[2 * l], ev[2 * l + 1]); attn_ms_accum += ms; }
    }
}

}  // namespace oa
