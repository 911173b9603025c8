/*
 * tests/kv_fp8_oracle.c — "mode 2" of the CPU oracle for the fp8 (e4m3) KV cache.  TEST INFRASTRUCTURE ONLY.
 *
 * Mode 2 is mode 1 (bf16-faithful) with one change: the KV cache holds e4m3(x * (1/s)) * s instead of x, where x is what mode 1 stores
 * (k after bias, bf16 round, RoPE and bf16 round; v after bias and bf16 round) and s is the layer's k or v scale.  To keep every other
 * operation identical to oracle/llama_ref.c, this file compiles that source unchanged and only intercepts the copies into a registered
 * model's cache: oa_ref_forward writes each new token's k and v rows with memcpy and attends to the cache afterwards, so the attention of
 * the same step already reads the quantised values.  Copies of 2 or 4 bytes (the bf16 bit casts) stay plain memcpy at compile time.
 *
 * e4m3 ("fn" variant): round to nearest even, saturating to +-448 (cvt.rn.satfinite.e4m3x2.f32), never a NaN code for finite input.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef struct { const float *k0, *k1, *v0, *v1; size_t layer_floats; int layers; float ks[256], vs[256]; } kv_fp8_reg;
static kv_fp8_reg g_reg[64];

__attribute__((visibility("default"))) uint8_t oa_ref_e4m3(float x) {
    const uint8_t sign = signbit(x) ? 0x80 : 0;
    if (isnan(x)) return sign | 0x7F;
    const float a = fabsf(x);
    if (a >= 448.0f) return sign | 0x7E;                         /* RNE of [448, 464) is 448 as well */
    if (a < 0.015625f) return sign | (uint8_t)rintf(a * 512.0f); /* subnormal step 2^-9; 8 steps = 2^-6 = code 0x08 */
    int E; frexpf(a, &E);                                         /* a = f * 2^E, f in [0.5, 1): exponent e = E - 1 */
    int e = E - 1, m = (int)rintf((ldexpf(a, -e) - 1.0f) * 8.0f);
    if (m == 8) { m = 0; ++e; }
    return sign | (uint8_t)(((e + 7) << 3) | m);
}
__attribute__((visibility("default"))) float oa_ref_e4m3_to_f32(uint8_t b) {
    const int e = (b >> 3) & 15, m = b & 7;
    if ((b & 0x7F) == 0x7F) return NAN;
    const float v = e == 0 ? ldexpf((float)m, -9) : ldexpf(1.0f + m / 8.0f, e - 7);
    return (b & 0x80) ? -v : v;
}

static void *kv_fp8_copy(void *d, const void *s, size_t n) {
    const float *p = (const float *)d;
    for (int i = 0; i < 64; ++i) {
        const kv_fp8_reg *r = &g_reg[i];
        if (!r->k0) continue;
        const int is_k = p >= r->k0 && p < r->k1, is_v = p >= r->v0 && p < r->v1;
        if (!is_k && !is_v) continue;
        const int layer = (int)((size_t)(p - (is_k ? r->k0 : r->v0)) / r->layer_floats % (size_t)r->layers);
        const float sc = is_k ? r->ks[layer] : r->vs[layer], inv = 1.0f / sc;
        const float *src = (const float *)s; float *dst = (float *)d;
        for (size_t j = 0; j < n / 4; ++j) dst[j] = oa_ref_e4m3_to_f32(oa_ref_e4m3(src[j] * inv)) * sc;
        return d;
    }
    return memcpy(d, s, n);
}
#define memcpy(d, s, n) (((n) <= 4) ? memcpy(d, s, n) : kv_fp8_copy(d, s, n))
#include "../oracle/llama_ref.c"
#undef memcpy

/* mode-2 model: a mode-1 oracle model whose cache copies are quantised with per-layer scales (k_scale / v_scale NULL: 1.0) */
REF_API ref_model *oa_ref2_create(const ref_config *cfg, int32_t max_pos, int32_t n_slots, const float *k_scale, const float *v_scale) {
    if (cfg->n_layers > 256) return NULL;
    for (int i = 0; i < 64; ++i) {
        kv_fp8_reg *r = &g_reg[i];
        if (r->k0) continue;
        ref_model *m = oa_ref_create(cfg, max_pos, n_slots, 1);
        const size_t kd = (size_t)cfg->n_kv_heads * cfg->head_dim, total = (size_t)n_slots * cfg->n_layers * max_pos * kd;
        r->layer_floats = (size_t)max_pos * kd; r->layers = cfg->n_layers;
        for (int l = 0; l < cfg->n_layers; ++l) { r->ks[l] = k_scale ? k_scale[l] : 1.0f; r->vs[l] = v_scale ? v_scale[l] : 1.0f; }
        r->k1 = m->kcache + total; r->v0 = m->vcache; r->v1 = m->vcache + total; r->k0 = m->kcache;
        return m;
    }
    return NULL;
}
REF_API void oa_ref2_destroy(ref_model *m) {
    for (int i = 0; i < 64; ++i) if (g_reg[i].k0 == m->kcache) memset(&g_reg[i], 0, sizeof g_reg[i]);
    oa_ref_destroy(m);
}
