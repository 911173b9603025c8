/*
 * tests/w8_fp8_oracle.c — "mode 3" of the CPU oracle for fp8 (e4m3) projection weights (W8A8).  TEST INFRASTRUCTURE ONLY.
 *
 * Mode 3 is mode 1 (or mode 0) with two changes on the seven per-layer projections (q, k, v, o, gate, up, down):
 *   - the weights are e4m3(w / s_w) * s_w, one scale per output row;
 *   - each row of a projection's input (xn, att, g = silu(gate) * up) is replaced by e4m3(x / s_x) * s_x, one scale per row.
 * The final norm output and the LM head are untouched.  Scales follow the row rule: s = the smallest power of two with max|row| <= 448 s
 * (all-zero row: 1; clamped to a normal fp32), so x / s and q * s are exact.
 *
 * oracle/llama_ref.c is compiled unchanged (through tests/kv_fp8_oracle.c, so mode 2's fp8 KV cache composes with this and the one e4m3
 * conversion, oa_ref_e4m3, is shared).  Its `linear` calls are routed to w8_linear by a macro that keys on the first argument's first
 * token: the definition (`const float *x`) becomes ref_linear, the REF_API wrapper (`x`) calls it, and the forward's calls (`xn`, `att`,
 * `g`) go to w8_linear.  A model that was not registered here, and the LM head of one that was, take ref_linear exactly as before.
 * With power-of-two scales e4m3(w / s) * s is a bf16 value, so a registered model's projections are quantised in place in its bf16 arrays;
 * a projection replaced through oa_ref3_set_weight (arbitrary positive scales, as FP8 checkpoints carry) is kept as an fp32 copy.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static void w8_linear(const void *m, const float *x, const uint16_t *W, const uint16_t *bias, float *y, int T, int K, int N);
#define linear(X, ...) W8LIN_##X, __VA_ARGS__)
#define W8LIN_const ref_linear(const
#define W8LIN_x ref_linear(x
#define W8LIN_xn w8_linear(m, xn
#define W8LIN_att w8_linear(m, att
#define W8LIN_g w8_linear(m, g
#include "kv_fp8_oracle.c"
#undef linear

/* the row rule on fp32 values */
REF_API float oa_ref_w8_scale(float amax) {
    uint32_t u; memcpy(&u, &amax, 4); u &= 0x7fffffffu;
    if (u == 0) return 1.0f;
    const int e = (int)(u >> 23);
    int k = e == 0 ? -126 : e - 135 + ((u & 0x7fffffu) > 0x600000u ? 1 : 0);
    if (k < -126) k = -126;
    const uint32_t sb = (uint32_t)(k + 127) << 23; float s; memcpy(&s, &sb, 4); return s;
}
/* one row -> e4m3 bytes + scale (either may be NULL) and the dequantised values (may alias x) */
REF_API float oa_ref_w8_row(const float *x, int n, uint8_t *q, float *deq) {
    float amax = 0.f;
    for (int i = 0; i < n; ++i) { const float a = fabsf(x[i]); if (a > amax) amax = a; }
    const float s = oa_ref_w8_scale(amax), inv = 1.0f / s;
    for (int i = 0; i < n; ++i) {
        const uint8_t b = oa_ref_e4m3(x[i] * inv);
        if (q) q[i] = b;
        if (deq) deq[i] = oa_ref_e4m3_to_f32(b) * s;
    }
    return s;
}

typedef struct { const ref_model *m; float **w[7]; } w8_reg;    /* w[kind][layer]: fp32 weights of wq..wd set by oa_ref3_set_weight, or NULL */
static w8_reg g_w8[64];

static w8_reg *w8_find(const void *m) {
    for (int i = 0; i < 64; ++i) if (g_w8[i].m && g_w8[i].m == m) return &g_w8[i];
    return NULL;
}
static uint16_t *w8_bits(const ref_model *m, int kind, int l) {
    uint16_t **a[7] = { m->wq, m->wk, m->wv, m->wo, m->wg, m->wu, m->wd };
    return a[kind][l];
}
static void w8_dims(const ref_model *m, int kind, int *N, int *K) {
    const int H = m->c.hidden, qd = m->c.n_heads * m->c.head_dim, kd = m->c.n_kv_heads * m->c.head_dim, F = m->c.ffn;
    const int n[7] = { qd, kd, kd, H, F, F, H }, k[7] = { H, H, H, qd, H, H, F };
    *N = n[kind]; *K = k[kind];
}

static void w8_linear(const void *mv, const float *x, const uint16_t *W, const uint16_t *bias, float *y, int T, int K, int N) {
    const ref_model *m = (const ref_model *)mv;
    w8_reg *r = w8_find(m);
    int proj = 0; const float *Wf = NULL;
    if (r) for (int l = 0; l < m->c.n_layers && !proj; ++l) for (int kind = 0; kind < 7; ++kind) if (W == w8_bits(m, kind, l)) { proj = 1; Wf = r->w[kind][l]; break; }
    if (!proj) { ref_linear(x, W, bias, y, T, K, N); return; }
    float *xq = (float *)malloc((size_t)T * K * sizeof(float));
    for (int t = 0; t < T; ++t) { memcpy(xq + (size_t)t * K, x + (size_t)t * K, (size_t)K * 4); oa_ref_w8_row(xq + (size_t)t * K, K, NULL, xq + (size_t)t * K); }
    if (!Wf) { ref_linear(xq, W, bias, y, T, K, N); free(xq); return; }
    #pragma omp parallel for schedule(static)
    for (int n = 0; n < N; ++n) {
        const float *w = Wf + (size_t)n * K;
        float b = bias ? bf16_to_f32(bias[n]) : 0.f;
        for (int t = 0; t < T; ++t) {
            const float *xr = xq + (size_t)t * K;
            float acc = 0.f;
            #pragma omp simd reduction(+:acc)
            for (int k = 0; k < K; ++k) acc += xr[k] * w[k];
            y[(size_t)t * N + n] = acc + b;
        }
    }
    free(xq);
}

/* Register m for W8A8: its projection weights are quantised in place with the row rule (exact in bf16). */
REF_API int oa_ref3_enable(ref_model *m) {
    for (int i = 0; i < 64; ++i) {
        w8_reg *r = &g_w8[i];
        if (r->m) continue;
        r->m = m;
        for (int kind = 0; kind < 7; ++kind) {
            r->w[kind] = (float **)calloc(m->c.n_layers, sizeof(float *));
            int N, K; w8_dims(m, kind, &N, &K);
            float *row = (float *)malloc((size_t)K * sizeof(float));
            for (int l = 0; l < m->c.n_layers; ++l) {
                uint16_t *b = w8_bits(m, kind, l);
                for (int n = 0; n < N; ++n) {
                    for (int k = 0; k < K; ++k) row[k] = bf16_to_f32(b[(size_t)n * K + k]);
                    oa_ref_w8_row(row, K, NULL, row);
                    for (int k = 0; k < K; ++k) b[(size_t)n * K + k] = f32_to_bf16(row[k]);
                }
            }
            free(row);
        }
        return 0;
    }
    return -1;
}
/* Replace one projection of a registered model by e4m3 bytes q [N, K] and per-row scales s [N] (any positive finite values). */
REF_API int oa_ref3_set_weight(ref_model *m, int32_t layer, int32_t kind, const uint8_t *q, const float *s) {
    w8_reg *r = w8_find(m);
    if (!r || layer < 0 || layer >= m->c.n_layers || kind < 0 || kind >= 7) return -1;
    int N, K; w8_dims(m, kind, &N, &K);
    if (!r->w[kind][layer]) r->w[kind][layer] = (float *)malloc((size_t)N * K * sizeof(float));
    float *w = r->w[kind][layer];
    for (int n = 0; n < N; ++n) for (int k = 0; k < K; ++k) w[(size_t)n * K + k] = oa_ref_e4m3_to_f32(q[(size_t)n * K + k]) * s[n];
    return 0;
}
/* fp32 copy of one registered projection [N, K] */
REF_API int oa_ref3_get_weight(ref_model *m, int32_t layer, int32_t kind, float *out) {
    w8_reg *r = w8_find(m);
    if (!r || layer < 0 || layer >= m->c.n_layers || kind < 0 || kind >= 7) return -1;
    int N, K; w8_dims(m, kind, &N, &K);
    if (r->w[kind][layer]) memcpy(out, r->w[kind][layer], (size_t)N * K * sizeof(float));
    else { const uint16_t *b = w8_bits(m, kind, layer); for (size_t j = 0; j < (size_t)N * K; ++j) out[j] = bf16_to_f32(b[j]); }
    return 0;
}
REF_API void oa_ref3_disable(ref_model *m) {
    w8_reg *r = w8_find(m);
    if (!r) return;
    for (int kind = 0; kind < 7; ++kind) { for (int l = 0; l < m->c.n_layers; ++l) free(r->w[kind][l]); free(r->w[kind]); }
    memset(r, 0, sizeof *r);
}
