// config.hpp — model architecture table, engine options and a minimal JSON reader for oa_engine_create().
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <map>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace oa {

// Flat JSON object reader: {"key": "str" | number | true | false | null, ...}.  Enough for engine configs.
class JsonFlat {
public:
    std::map<std::string, std::string> kv;   // raw values (strings unescaped)
    static JsonFlat parse(const std::string& s) {
        JsonFlat j; size_t i = 0;
        auto ws = [&]() { while (i < s.size() && (s[i] == ' ' || s[i] == '\n' || s[i] == '\t' || s[i] == '\r')) ++i; };
        auto str = [&]() -> std::string {
            if (s[i] != '"') throw std::runtime_error("config json: expected string");
            ++i; std::string o;
            while (i < s.size() && s[i] != '"') {
                if (s[i] == '\\' && i + 1 < s.size()) { ++i; char c = s[i]; o += (c == 'n' ? '\n' : c == 't' ? '\t' : c); }
                else o += s[i];
                ++i;
            }
            if (i >= s.size()) throw std::runtime_error("config json: unterminated string");
            ++i; return o;
        };
        ws(); if (i >= s.size() || s[i] != '{') throw std::runtime_error("config json: expected object");
        ++i; ws();
        if (i < s.size() && s[i] == '}') return j;
        while (true) {
            ws(); std::string k = str(); ws();
            if (i >= s.size() || s[i] != ':') throw std::runtime_error("config json: expected ':'");
            ++i; ws();
            std::string v;
            if (s[i] == '"') v = str();
            else { size_t b = i; while (i < s.size() && s[i] != ',' && s[i] != '}' && s[i] != ' ' && s[i] != '\n') ++i; v = s.substr(b, i - b); }
            j.kv[k] = v; ws();
            if (i < s.size() && s[i] == ',') { ++i; continue; }
            if (i < s.size() && s[i] == '}') break;
            throw std::runtime_error("config json: expected ',' or '}'");
        }
        return j;
    }
    bool has(const std::string& k) const { return kv.count(k) && kv.at(k) != "null"; }
    std::string s(const std::string& k, const std::string& d) const { return has(k) ? kv.at(k) : d; }
    double f(const std::string& k, double d) const {
        if (!has(k)) return d;
        const std::string& v = kv.at(k);
        if (v == "true") return 1; if (v == "false") return 0;
        return std::strtod(v.c_str(), nullptr);
    }
    int64_t i(const std::string& k, int64_t d) const { return has(k) ? (int64_t)std::llround(f(k, (double)d)) : d; }
};

struct ModelConfig {
    std::string name = "custom";
    int hidden = 0, n_layers = 0, n_heads = 0, n_kv_heads = 0, head_dim = 0, ffn = 0, vocab = 0;
    int tie_embeddings = 0, qkv_bias = 0, rope_scaling = 0, norm_random = 0;
    float rope_theta = 500000.f, rms_eps = 1e-5f;
    float rope_factor = 32.f, rope_low_freq = 1.f, rope_high_freq = 4.f; int rope_orig_ctx = 8192;
    float init_std = 0.02f;
    uint64_t seed = 1234;
    std::string chat_template = "llama3";   // or "chatml"

    int q_dim() const { return n_heads * head_dim; }
    int kv_dim() const { return n_kv_heads * head_dim; }
    int qkv_dim() const { return q_dim() + 2 * kv_dim(); }
    std::string kv_cache_dtype = "bf16";    // paged KV cache storage: "bf16" or "fp8_e4m3" (one byte per element, per-layer K / V scales)
    bool kv_fp8() const { return kv_cache_dtype == "fp8_e4m3"; }
    int kv_elem_bytes() const { return kv_fp8() ? 1 : 2; }
    size_t kv_bytes_per_token() const { return (size_t)2 * n_layers * kv_dim() * kv_elem_bytes(); }
    // projection weights (qkv, o, gate/up, down): "bf16", or "fp8_e4m3" (one byte per element plus one fp32 scale per output row; W8A8 GEMMs
    // with per-token activation scales).  Embedding, LM head, norms and biases stay bf16.
    std::string weight_dtype = "bf16";
    bool w_fp8() const { return weight_dtype == "fp8_e4m3"; }
    double decode_weight_bytes() const {   // W_dec of SURVEY.md §8d: all layers + final norm + lm_head
        const double proj = (double)qkv_dim() * hidden + (double)hidden * q_dim() + 3.0 * ffn * hidden;
        const double rows = (double)qkv_dim() + hidden + 2.0 * ffn + hidden;            // one fp32 scale per output row (fp8)
        const double other = 2.0 * hidden + (qkv_bias ? qkv_dim() : 0);
        if (w_fp8()) return (proj + 4.0 * rows + 2.0 * other) * n_layers + 2.0 * (hidden + (double)vocab * hidden);
        return 2.0 * ((proj + other) * n_layers + hidden + (double)vocab * hidden);
    }
};

// public architectures (SURVEY.md §8d); oracle/oracle.py PRESETS is the test-side copy
inline bool preset_model(const std::string& n, ModelConfig& c) {
    c.name = n;
    if (n == "llama-3.2-1b") { c.hidden = 2048; c.n_layers = 16; c.n_heads = 32; c.n_kv_heads = 8; c.head_dim = 64; c.ffn = 8192; c.vocab = 128256; c.tie_embeddings = 1; c.rope_scaling = 1; return true; }
    if (n == "llama-3-8b") { c.hidden = 4096; c.n_layers = 32; c.n_heads = 32; c.n_kv_heads = 8; c.head_dim = 128; c.ffn = 14336; c.vocab = 128256; return true; }
    if (n == "qwen2.5-32b") { c.hidden = 5120; c.n_layers = 64; c.n_heads = 40; c.n_kv_heads = 8; c.head_dim = 128; c.ffn = 27648; c.vocab = 152064; c.qkv_bias = 1; c.rope_theta = 1e6f; c.rms_eps = 1e-6f; c.chat_template = "chatml"; return true; }
    if (n == "llama-3-70b") { c.hidden = 8192; c.n_layers = 80; c.n_heads = 64; c.n_kv_heads = 8; c.head_dim = 128; c.ffn = 28672; c.vocab = 128256; return true; }
    return false;
}

struct EngineOptions {
    int device = 0;
    double kv_gb = -1;            // < 0: use what is free after weights minus a reserve
    int num_pages = -1;           // overrides kv_gb
    int max_batch = 256;          // concurrently running sequences
    int max_seq_len = 4096;       // prompt + completion
    int max_step_tokens = 8192;   // token budget of one prefill forward
    int max_queue = 4096;         // waiting requests beyond this -> 429
    int bn_qkv = 0, bn_o = 0, bn_gu = 0, bn_down = 0, bn_lm = 0;   // GEMM N-tile overrides (0 = heuristic)
    int attn_ctas = 0;            // decode attention CTA count override (0 = 2 per SM)
    int streamk = 1;              // decode (T <= 128) projections through the persistent stream-K GEMM
    int sk_bn = 128, sk_ctas = 0; // its N tile (128: half the partial traffic of 256, and a 64 x 128 fp32 fragment per consumer warpgroup) and CTA count (0 = one per SM)
    int sk_max_rows = 128;        // batches up to this many rows use stream-K (256 = two row tiles, opt-in)
    int sk_fuse_swiglu = 1;       // gate/up projection: the CTA holding a tile's first k-block adds the other pieces and writes silu(gate)*up from its accumulator (no SwiGLU kernel)
    int sk_fuse_epi = 0;          // bitmask — 1: qkv finishes bias + RoPE + paged-KV write, 2: o, 4: down finish the residual add inside the stream-K GEMM (the CTA holding a tile's first k-block; a norm-only kernel follows o / down).
                                  // Bit-identical to the consumers; off by default: few tiles cut into 4-5 pieces each make the finishers a serial tail
    int sk_clusterk = 0;          // bitmask — 1: qkv, 2: o, 4: down as a cluster split-K GEMM with DSMEM reduction and the epilogue (RoPE + KV write / residual) inside (gemm_clusterk.cu), where the shape fills >= 80 % of the SMs
    int sk_clusterk_min_fill = 80; // ... and only where n_tiles x cluster size covers at least this percentage of the SMs (tests: 0)
    int sk_l2_prefetch_kb = 0;    // per-CTA weight KB prefetched into L2 ahead of the dependency wait (0 = off)
    int sk_bn_qkv = 0, sk_bn_o = 0, sk_bn_gu = 0, sk_bn_down = 0;   // per-projection overrides (0 = sk_bn)
    int start_thread = 1;
    std::string model_aliases;    // other model names this engine answers to, comma separated ("*" = any): the reference sends currentModel or "gpt-4" (execute.go:168-171)
    std::string weights;          // path of a Hugging Face *.safetensors file or shard directory (empty: seeded random init)
    int prefix_cache = 1;         // reuse KV pages of shared prompt prefixes across requests (the ReAct loop resends its history)
    int json_mode = 0;            // 1: every chat completion is grammar-forced to parse as tools.ToolPrompt (tool.go:29-38)
    std::string tokenizer;             // path of a Hugging Face tokenizer.json (byte-level BPE, Llama-3 / Qwen2.5 format); empty = synthetic byte-level ids
    int prefill_batch_tokens = 2048;   // while sequences are decoding, new requests wait until this many uncached prompt tokens are queued ...
    int prefill_max_wait_ms = 20;      // ... or the oldest has waited this long: one weight pass then prefills several arrivals (0 tokens = admit at once)
    int mixed_steps = 1;               // decoding sequences ride along in prefill steps (decode attention for their rows, prefill attention for the chunks) instead of stalling for every arrival's weight pass; 0 = prefill-first steps only
    int react_tool_steps = 3;     // json_mode: conversations with fewer assistant turns than this get a tool call, later ones a final answer
    int tp = 1, tp_rank = 0;      // tensor parallel degree / this process's rank (one process per GPU)
    std::string tp_shm = "/oa_tp"; // POSIX shm name shared by the ranks of one TP group
    int tp_ar_bf16 = 1;            // decode all-reduce on bf16 partials (half the NVLink bytes; the prefill path always exchanged bf16); 0 = fp32 partials
    int tp_nvls = 0;               // 1: decode all-reduce inside the NVLink switch (multimem.ld_reduce / multimem.st on a multicast buffer, tp_nvls.cpp) when every rank can set it up.  Built, parity-green,
                                   // opt-in: three dependent cross-GPU latencies on the critical path instead of the peer-memory one-shot's one
    int tp_two_shot_rows = 1024;   // prefill chunks of at least this many rows use the two-shot all-reduce (reduce-scatter + all-gather: 2(t-1)/t instead of (t-1) partials' bytes per rank); smaller ones the one-shot
    uint64_t tp_nonce = 0;         // per-launch id shared by the ranks (e.g. the rendezvous port + a timestamp): followers ignore segments of other launches (0 = not checked)
};

inline void parse_config(const std::string& json, ModelConfig& m, EngineOptions& o) {
    JsonFlat j = JsonFlat::parse(json);
    std::string name = j.s("model", "custom");
    if (!preset_model(name, m)) m.name = name;
    auto I = [&](const char* k, int& v) { v = (int)j.i(k, v); };
    auto F = [&](const char* k, float& v) { v = (float)j.f(k, v); };
    I("hidden", m.hidden); I("n_layers", m.n_layers); I("n_heads", m.n_heads); I("n_kv_heads", m.n_kv_heads);
    I("head_dim", m.head_dim); I("ffn", m.ffn); I("vocab", m.vocab); I("tie_embeddings", m.tie_embeddings);
    I("qkv_bias", m.qkv_bias); I("rope_scaling", m.rope_scaling); I("norm_random", m.norm_random);
    F("rope_theta", m.rope_theta); F("rms_eps", m.rms_eps); F("rope_factor", m.rope_factor);
    F("rope_low_freq", m.rope_low_freq); F("rope_high_freq", m.rope_high_freq); I("rope_orig_ctx", m.rope_orig_ctx);
    F("init_std", m.init_std);
    m.seed = (uint64_t)j.i("seed", (int64_t)m.seed);
    m.chat_template = j.s("template", m.chat_template);
    m.kv_cache_dtype = j.s("kv_cache_dtype", m.kv_cache_dtype);
    m.weight_dtype = j.s("weight_dtype", m.weight_dtype);
    I("device", o.device); o.kv_gb = j.f("kv_gb", o.kv_gb); I("num_pages", o.num_pages); I("max_batch", o.max_batch);
    I("max_seq_len", o.max_seq_len); I("max_step_tokens", o.max_step_tokens); I("max_queue", o.max_queue);
    I("bn_qkv", o.bn_qkv); I("bn_o", o.bn_o); I("bn_gu", o.bn_gu); I("bn_down", o.bn_down); I("bn_lm", o.bn_lm);
    I("attn_ctas", o.attn_ctas); I("streamk", o.streamk); I("sk_bn", o.sk_bn); I("sk_ctas", o.sk_ctas); I("sk_l2_prefetch_kb", o.sk_l2_prefetch_kb); I("sk_max_rows", o.sk_max_rows); I("sk_fuse_swiglu", o.sk_fuse_swiglu); I("sk_fuse_epi", o.sk_fuse_epi); I("sk_clusterk", o.sk_clusterk); I("sk_clusterk_min_fill", o.sk_clusterk_min_fill); I("sk_bn_qkv", o.sk_bn_qkv); I("sk_bn_o", o.sk_bn_o); I("sk_bn_gu", o.sk_bn_gu); I("sk_bn_down", o.sk_bn_down); I("start_thread", o.start_thread); o.weights = j.s("weights", o.weights); o.model_aliases = j.s("model_aliases", o.model_aliases); o.tokenizer = j.s("tokenizer", o.tokenizer); I("prefix_cache", o.prefix_cache); I("json_mode", o.json_mode); I("react_tool_steps", o.react_tool_steps); I("prefill_batch_tokens", o.prefill_batch_tokens); I("mixed_steps", o.mixed_steps); I("prefill_max_wait_ms", o.prefill_max_wait_ms); I("tp", o.tp); I("tp_rank", o.tp_rank); I("tp_ar_bf16", o.tp_ar_bf16); I("tp_nvls", o.tp_nvls); I("tp_two_shot_rows", o.tp_two_shot_rows); o.tp_shm = j.s("tp_shm", o.tp_shm); o.tp_nonce = (uint64_t)j.i("tp_nonce", (int64_t)o.tp_nonce);
    if (m.hidden <= 0 || m.n_layers <= 0 || m.n_heads <= 0 || m.n_kv_heads <= 0 || m.ffn <= 0 || m.vocab <= 0)
        throw std::runtime_error("unknown model '" + name + "' and no explicit dimensions given");
    if (m.head_dim != 64 && m.head_dim != 128) throw std::runtime_error("head_dim must be 64 or 128");
    if (m.n_heads % m.n_kv_heads != 0 || m.n_heads / m.n_kv_heads > 8) throw std::runtime_error("GQA group must divide n_heads and be <= 8");
    if (m.hidden % 64 || m.ffn % 64 || m.vocab % 8) throw std::runtime_error("hidden/ffn must be multiples of 64, vocab of 8");
    if (m.chat_template != "llama3" && m.chat_template != "chatml") throw std::runtime_error("template must be llama3 or chatml");
    if (m.kv_cache_dtype != "bf16" && m.kv_cache_dtype != "fp8_e4m3") throw std::runtime_error("kv_cache_dtype must be bf16 or fp8_e4m3");
    if (m.weight_dtype != "bf16" && m.weight_dtype != "fp8_e4m3") throw std::runtime_error("weight_dtype must be bf16 or fp8_e4m3");
    if (m.w_fp8() && o.tp != 1) throw std::runtime_error("weight_dtype fp8_e4m3 needs tp = 1 (row-parallel shards would need whole-row weight scales)");
    if (m.w_fp8() && o.sk_clusterk != 0) throw std::runtime_error("weight_dtype fp8_e4m3 needs sk_clusterk = 0 (the cluster split-K GEMM is bf16 only)");
    if (o.max_seq_len % 64) o.max_seq_len = (o.max_seq_len + 63) / 64 * 64;
    if (o.tp < 1 || o.tp > 8 || o.tp_rank < 0 || o.tp_rank >= o.tp) throw std::runtime_error("tp must be 1..8 and 0 <= tp_rank < tp");
    if (o.tp > 1 && (m.n_kv_heads % o.tp || m.n_heads % o.tp || (m.ffn / o.tp) % 64 || m.ffn % o.tp || (m.vocab / o.tp) % 8 || m.vocab % o.tp))
        throw std::runtime_error("tp must divide n_heads, n_kv_heads, ffn (in multiples of 64) and vocab (in multiples of 8)");
}

}  // namespace oa
