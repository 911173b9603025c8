// checkpoint.hpp — host half of the Hugging Face checkpoint loader (Llama / Qwen2 naming): which rows of which tensors make up each
// matrix this tensor-parallel rank holds, and their assembly into bf16 rows or e4m3 bytes + fp32 row scales.  No CUDA calls: the device
// model uploads what this returns.
#pragma once
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "common.cuh"
#include "config.hpp"
#include "safetensors.hpp"

namespace oa {

inline float f16_bits_to_f32(uint16_t hb) {
    const uint32_t h = hb, sign = (h & 0x8000u) << 16, e = (h >> 10) & 31, m = h & 1023; uint32_t f;
    if (e == 0) { if (m == 0) f = sign; else { int sh = 0; uint32_t mm = m; while (!(mm & 1024)) { mm <<= 1; ++sh; } f = sign | ((uint32_t)(113 - sh) << 23) | ((mm & 1023) << 13); } }
    else if (e == 31) f = sign | 0x7f800000u | (m << 13);
    else f = sign | ((e + 112) << 23) | (m << 13);
    float x; std::memcpy(&x, &f, 4); return x;
}

// element j of an F32 / BF16 / F16 scale tensor `name`; a scale must be finite and > 0
inline float ckpt_scale(const StTensor& t, int64_t j, const std::string& name) {
    float v;
    if (t.dtype == "F32") std::memcpy(&v, t.data + 4 * j, 4);
    else if (t.dtype == "BF16") { uint16_t b; std::memcpy(&b, t.data + 2 * j, 2); const uint32_t u = (uint32_t)b << 16; std::memcpy(&v, &u, 4); }
    else if (t.dtype == "F16") { uint16_t b; std::memcpy(&b, t.data + 2 * j, 2); v = f16_bits_to_f32(b); }
    else throw std::runtime_error("checkpoint tensor " + name + " has unsupported dtype " + t.dtype);
    if (!std::isfinite(v) || v <= 0.f) throw std::runtime_error("checkpoint tensor " + name + " must be finite and > 0");
    return v;
}

// fp8 KV cache scales (compressed-tensors / vLLM naming): model.layers.{l}.self_attn.k_scale / v_scale, shape [] or [1], F32 / BF16 / F16,
// finite and > 0, present for every layer or for none (then 1.0)
inline void load_kv_scales(const SafeTensors& st, int L, std::vector<float>& ks, std::vector<float>& vs) {
    auto scalar = [&](const std::string& name) -> float {
        const StTensor& t = st.get(name);
        if (!(t.shape.empty() || (t.shape.size() == 1 && t.shape[0] == 1))) throw std::runtime_error("checkpoint tensor " + name + " must have shape [] or [1]");
        return ckpt_scale(t, 0, name);
    };
    int nk = 0, nv = 0;
    for (int l = 0; l < L; ++l) {
        const std::string p = "model.layers." + std::to_string(l) + ".self_attn.";
        nk += st.has(p + "k_scale"); nv += st.has(p + "v_scale");
    }
    if (nk == 0 && nv == 0) return;
    for (const auto& c : {std::make_pair("k_scale", nk), std::make_pair("v_scale", nv)})
        if (c.second != L) throw std::runtime_error("checkpoint has self_attn." + std::string(c.first) + " for " + std::to_string(c.second) + " of " +
                                                    std::to_string(L) + " layers: KV cache scales must be given for every layer or for none");
    for (int l = 0; l < L; ++l) {
        const std::string p = "model.layers." + std::to_string(l) + ".self_attn.";
        ks[l] = scalar(p + "k_scale"); vs[l] = scalar(p + "v_scale");
    }
}

// One piece of a device matrix: rows [row0, row0 + rows) x columns [col0, col0 + cols) of the logical [R, C] checkpoint tensor `name`
// (a vector is [1, C]).
struct CkptPart { std::string name; int64_t R, C, row0, rows, col0, cols; };
// A device matrix as its physical rows: the parts' rows one after the other, or, for gate/up, alternating blocks of 16 rows of parts[0]
// and parts[1] (the layout the SwiGLU epilogues read).
struct CkptRows {
    std::vector<CkptPart> parts; bool gate_up = false;
    template <class Fn> void for_each_row(Fn fn) const {      // fn(part index, row of the part's range), in physical row order
        if (gate_up) {
            for (int64_t b = 0; b < parts[0].rows / 16; ++b)
                for (int w = 0; w < 32; ++w) fn(w >> 4, b * 16 + (w & 15));
            return;
        }
        for (size_t p = 0; p < parts.size(); ++p)
            for (int64_t i = 0; i < parts[p].rows; ++i) fn((int)p, i);
    }
};

// What one tensor-parallel rank loads: column-parallel q|k|v and gate|up take row shards, row-parallel o and down column shards of the
// logical tensors, the vocab-parallel LM head a row shard; embedding and norms are whole.
struct CkptLayerRows { CkptRows qkv, o, gu, down, ln1, ln2, bqkv; };
struct CkptShard {
    CkptRows embed, norm, lm_head; std::vector<CkptLayerRows> layers;
    CkptShard(const SafeTensors& st, const ModelConfig& c, int tp, int rank) {
        const int64_t H = c.hidden, V_l = c.vocab / tp, qd = c.q_dim() / tp, kd = c.kv_dim() / tp, F = c.ffn / tp, r = rank;
        embed.parts = {{"model.embed_tokens.weight", c.vocab, H, 0, c.vocab, 0, H}};
        norm.parts = {{"model.norm.weight", 1, H, 0, 1, 0, H}};
        lm_head.parts = {{st.has("lm_head.weight") ? "lm_head.weight" : "model.embed_tokens.weight", c.vocab, H, r * V_l, V_l, 0, H}};
        for (int l = 0; l < c.n_layers; ++l) {
            const std::string p = "model.layers." + std::to_string(l) + ".";
            CkptLayerRows y;
            y.qkv.parts = {{p + "self_attn.q_proj.weight", c.q_dim(), H, r * qd, qd, 0, H}, {p + "self_attn.k_proj.weight", c.kv_dim(), H, r * kd, kd, 0, H},
                           {p + "self_attn.v_proj.weight", c.kv_dim(), H, r * kd, kd, 0, H}};
            y.o.parts = {{p + "self_attn.o_proj.weight", H, c.q_dim(), 0, H, r * qd, qd}};
            y.gu.parts = {{p + "mlp.gate_proj.weight", c.ffn, H, r * F, F, 0, H}, {p + "mlp.up_proj.weight", c.ffn, H, r * F, F, 0, H}};
            y.gu.gate_up = true;
            y.down.parts = {{p + "mlp.down_proj.weight", H, c.ffn, 0, H, r * F, F}};
            y.ln1.parts = {{p + "input_layernorm.weight", 1, H, 0, 1, 0, H}};
            y.ln2.parts = {{p + "post_attention_layernorm.weight", 1, H, 0, 1, 0, H}};
            if (c.qkv_bias)
                y.bqkv.parts = {{p + "self_attn.q_proj.bias", 1, c.q_dim(), 0, 1, r * qd, qd}, {p + "self_attn.k_proj.bias", 1, c.kv_dim(), 0, 1, r * kd, kd},
                                {p + "self_attn.v_proj.bias", 1, c.kv_dim(), 0, 1, r * kd, kd}};
            layers.push_back(std::move(y));
        }
    }
};

// Every tensor must have exactly the logical shape [R, C] (vectors: [C]) this model configuration implies — a transposed, truncated or
// wrong-config (hidden / ffn / heads / vocab) checkpoint is refused with a message instead of being read out of bounds.  F8_E4M3 is
// accepted for projection weights under weight_dtype fp8_e4m3 only.
inline const StTensor& ckpt_part(const SafeTensors& st, const CkptPart& p, bool w8) {
    const StTensor& t = st.get(p.name);
    const bool ok = (t.shape.size() == 2 && t.shape[0] == p.R && t.shape[1] == p.C) || (p.R == 1 && t.shape.size() == 1 && t.shape[0] == p.C);
    if (!ok) {
        std::string got = "["; for (size_t i = 0; i < t.shape.size(); ++i) got += (i ? ", " : "") + std::to_string(t.shape[i]); got += "]";
        throw std::runtime_error("checkpoint tensor " + p.name + " has shape " + got + ", this model needs [" + (p.R == 1 ? "" : std::to_string(p.R) + ", ") + std::to_string(p.C) + "]");
    }
    if (p.row0 < 0 || p.col0 < 0 || p.row0 + p.rows > p.R || p.col0 + p.cols > p.C) throw std::runtime_error("checkpoint slice out of range for " + p.name);
    const bool proj = p.name.size() > 12 && p.name.compare(p.name.size() - 12, 12, "_proj.weight") == 0;     // q/k/v/o/gate/up/down
    if (proj && t.dtype == "F8_E4M3") {
        if (!w8) throw std::runtime_error("checkpoint tensor " + p.name + " is F8_E4M3: fp8 projection weights need weight_dtype fp8_e4m3");
        return t;
    }
    if (t.dtype != "BF16" && t.dtype != "F16" && t.dtype != "F32") throw std::runtime_error("checkpoint tensor " + p.name + " has unsupported dtype " + t.dtype);
    return t;       // SafeTensors already verified bytes == prod(shape) * sizeof(dtype)
}

// Checks every part; true when all are F8_E4M3 (compressed-tensors "FP8" checkpoints), false when none is.  One matrix takes one kind.
inline bool ckpt_is_f8(const SafeTensors& st, const CkptRows& m, bool w8) {
    size_t n_f8 = 0;
    for (const CkptPart& p : m.parts) n_f8 += ckpt_part(st, p, w8).dtype == "F8_E4M3";
    if (n_f8 != 0 && n_f8 != m.parts.size())
        throw std::runtime_error("checkpoint tensor " + m.parts[0].name + ": the parts of one fused projection (q/k/v, gate/up) must all be F8_E4M3 or none");
    return n_f8 != 0;
}

// BF16 / F16 / F32 parts -> bf16 bits, the physical rows back to back (each row its part's cols wide)
inline void ckpt_bf16(const SafeTensors& st, const CkptRows& m, std::vector<uint16_t>& out) {
    std::vector<const StTensor*> ts;
    size_t n = 0;
    for (const CkptPart& p : m.parts) { ts.push_back(&ckpt_part(st, p, false)); n += (size_t)p.rows * p.cols; }
    out.resize(n);
    uint16_t* dst = out.data();
    m.for_each_row([&](int pi, int64_t i) {
        const CkptPart& p = m.parts[pi]; const StTensor& t = *ts[pi];
        const size_t at = (size_t)(p.row0 + i) * p.C + p.col0;
        if (t.dtype == "BF16") std::memcpy(dst, reinterpret_cast<const uint16_t*>(t.data) + at, (size_t)p.cols * 2);
        else if (t.dtype == "F32") { const float* s = reinterpret_cast<const float*>(t.data) + at; for (int64_t j = 0; j < p.cols; ++j) dst[j] = f32_to_bf16_bits(s[j]); }
        else { const uint16_t* s = reinterpret_cast<const uint16_t*>(t.data) + at; for (int64_t j = 0; j < p.cols; ++j) dst[j] = f32_to_bf16_bits(f16_bits_to_f32(s[j])); }
        dst += p.cols;
    });
}

// F8_E4M3 parts -> their bytes and one fp32 scale per physical row from `<name>_scale`: per row ([R, 1] / [R]) or per tensor ([] / [1]).
// Static activation scales (`input_scale`) are not read: activations are quantised per token at run time.
inline void ckpt_f8(const SafeTensors& st, const CkptRows& m, std::vector<uint8_t>& q, std::vector<float>& s) {
    std::vector<const StTensor*> ts, ss; std::vector<bool> per_row;
    size_t n = 0, rows = 0;
    for (const CkptPart& p : m.parts) {
        ts.push_back(&ckpt_part(st, p, true));
        const std::string sn = p.name + "_scale";
        if (!st.has(sn)) throw std::runtime_error("checkpoint tensor " + p.name + " is F8_E4M3 but " + sn + " is missing");
        const StTensor& t = st.get(sn);
        const bool pr = (t.shape.size() == 2 && t.shape[0] == p.R && t.shape[1] == 1) || (t.shape.size() == 1 && t.shape[0] == p.R);
        const bool pt = t.shape.empty() || (t.shape.size() == 1 && t.shape[0] == 1) || (t.shape.size() == 2 && t.shape[0] == 1 && t.shape[1] == 1);
        if (!pr && !pt) throw std::runtime_error("checkpoint tensor " + sn + " must have shape [" + std::to_string(p.R) + ", 1], [" + std::to_string(p.R) + "], [] or [1]");
        ss.push_back(&t); per_row.push_back(pr);
        n += (size_t)p.rows * p.cols; rows += (size_t)p.rows;
    }
    q.resize(n); s.resize(rows);
    uint8_t* dst = q.data(); float* sd = s.data();
    m.for_each_row([&](int pi, int64_t i) {
        const CkptPart& p = m.parts[pi];
        std::memcpy(dst, ts[pi]->data + (size_t)(p.row0 + i) * p.C + p.col0, (size_t)p.cols);
        *sd++ = ckpt_scale(*ss[pi], per_row[pi] ? p.row0 + i : 0, p.name + "_scale");
        dst += p.cols;
    });
}

}  // namespace oa
