/*
 * opsagent_b200.h — C ABI of the H100-native local chat-completion engine.
 *
 * This is the drop-in boundary behind OpsAgent's LLM seam.  The reference has no FFI for this path;
 * its seam is the Go method
 *     func (c *OpenAIClient) Chat(model string, maxTokens int, prompts []openai.ChatCompletionMessage) (string, error)
 * (reference pkg/llms/openai.go:69-104), which today POSTs {model, messages, max_tokens, temperature}
 * to a remote /chat/completions server.  The entry points below are what a `local-cuda` provider binds
 * through cgo instead (INTEGRATION.md shows the Go side).  Plain C types only; no exceptions cross the
 * boundary; every function is safe to call from any thread.
 *
 * Return codes mirror the HTTP statuses the reference's retry loop already understands
 * (pkg/llms/openai.go:85-101): 0 ok; 400 bad request (fails fast); 429 queue/KV full (caller backs
 * off 1,2,4,8,16 s and retries); 500 device or internal fault (retried likewise).
 */
#ifndef OPSAGENT_B200_H
#define OPSAGENT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define OA_API __attribute__((visibility("default")))
#else
#define OA_API
#endif

#define OA_OK 0
#define OA_ERR_BAD_REQUEST 400
#define OA_ERR_TIMEOUT 408
#define OA_ERR_OVERLOADED 429
#define OA_ERR_INTERNAL 500

typedef struct oa_engine oa_engine; /* opaque, process-global, thread-safe */

/* replaces openai.ChatCompletionMessage{Role, Content} (go-openai v1.38.0; used at pkg/llms/openai.go:69) */
typedef struct {
    const char* role;    /* "system" | "user" | "assistant"; UTF-8, NUL-terminated, caller-owned */
    const char* content; /* UTF-8, NUL-terminated, caller-owned */
} oa_msg;

/* replaces openai.ChatCompletionRequest as built at pkg/llms/openai.go:70-75 */
typedef struct {
    const char* model;     /* must name the loaded model (or be empty/NULL) — else 400 */
    const oa_msg* msgs;
    int32_t n_msgs;
    int32_t max_tokens;    /* completion budget (8192 from pkg/handlers/execute.go:205) */
    float temperature;     /* the reference always sends SmallestNonzeroFloat32: greedy. Values > 1e-3 -> 400 */
    uint64_t seed;         /* unused under greedy decoding; kept for ABI stability */
    uint32_t flags;        /* OA_FLAG_* */
    const char* functions; /* OA_FLAG_JSON_FUNCTION: "name:param,name:param" — the functions the request's `tools` array offers */
} oa_chat_req;

#define OA_FLAG_IGNORE_EOS 1u /* throughput runs: always generate exactly max_tokens tokens */
#define OA_FLAG_JSON_TOOLCALL 2u /* force the completion to parse as tools.ToolPrompt (pkg/tools/tool.go:29-38) with an action from the
                                  * tool registry (tool.go:20-26) and an empty final_answer: one ReAct tool-call step */
#define OA_FLAG_JSON_FUNCTION 8u /* OpenAI function calling (swarm-go flows, pkg/workflows/swarm.go:14-78): the completion is
                                  * {"name":"<offered function>","arguments":{"<its parameter>":"..."}} */
#define OA_FLAG_JSON_TEXT 16u    /* one bounded line of printable text (10..200 bytes), newline-terminated */
#define OA_FLAG_JSON_FINAL 4u    /* same schema, empty action, final_answer of >= 10 bytes (not a placeholder per simple.go:640-654) */

/* replaces resp.Choices[0].Message.Content (+ usage) at pkg/llms/openai.go:82 */
typedef struct {
    char* content;         /* engine-owned, NUL-terminated, may contain embedded NULs: use content_len */
    int32_t content_len;
    int32_t prompt_tokens, completion_tokens;
    int32_t finish_reason; /* 0 stop (EOS), 1 length */
    int32_t* token_ids;    /* completion token ids (engine-owned), length completion_tokens */
} oa_chat_resp;

/* config_json: {"model":"llama-3-8b"|"llama-3.2-1b"|"qwen2.5-32b"|"llama-3-70b"|custom dims..., "seed":1234,
 *  "device":0, "kv_gb":100, "max_batch":128, "max_seq_len":4096, "max_step_tokens":8192,
 *  "kv_cache_dtype":"bf16"|"fp8_e4m3", "weight_dtype":"bf16"|"fp8_e4m3", ...} — see DESIGN.md */
OA_API int oa_engine_create(const char* config_json, oa_engine** out);
OA_API void oa_engine_destroy(oa_engine*);
/* tensor-parallel groups (config "tp": t, "tp_rank": r, "tp_shm": name; one process per GPU): rank 0 is the engine callers talk
 * to; every other rank calls oa_engine_serve(), which replays the leader's steps and returns when the leader is destroyed */
OA_API int oa_engine_serve(oa_engine*);

/* blocking completion — what (*LocalCUDAClient).Chat calls; replaces CreateChatCompletion (openai.go:79) */
OA_API int oa_chat_complete(oa_engine*, const oa_chat_req*, oa_chat_resp* out);
/* non-blocking pair for callers that must not pin an OS thread per request (Go: submit, then wait) */
OA_API int oa_chat_submit(oa_engine*, const oa_chat_req*, uint64_t* ticket);
OA_API int oa_chat_wait(oa_engine*, uint64_t ticket, int32_t timeout_ms, oa_chat_resp* out);
/* abandon a submitted request (wait timed out, caller's context cancelled): frees its queue slot / KV pages; the ticket dies */
OA_API int oa_chat_cancel(oa_engine*, uint64_t ticket);
/* the same pair with the error text copied into a caller buffer instead of the thread-local oa_last_error(): what the cgo binding
 * uses, so that goroutines need not be pinned to an OS thread with runtime.LockOSThread for the duration of a Chat */
OA_API int oa_chat_submit_ex(oa_engine*, const oa_chat_req*, uint64_t* ticket, char* errbuf, size_t errcap);
OA_API int oa_chat_wait_ex(oa_engine*, uint64_t ticket, int32_t timeout_ms, oa_chat_resp* out, char* errbuf, size_t errcap);
OA_API void oa_free_resp(oa_chat_resp*);

/* same pair on raw token ids (bench + parity tests; bypasses the chat template) */
OA_API int oa_tokens_submit(oa_engine*, const int32_t* prompt, int32_t n_prompt, int32_t max_tokens, uint32_t flags, uint64_t* ticket);

/* tokenizer-accurate counting for pkg/llms/tokens.go:60 NumTokensFromMessages / :128 ConstrictPrompt */
OA_API int oa_count_tokens(oa_engine*, const oa_msg* msgs, int32_t n_msgs, int32_t* out_tokens);
/* chat template + tokenizer only: writes up to cap ids, returns total count in *n_out */
OA_API int oa_apply_chat_template(oa_engine*, const oa_msg* msgs, int32_t n_msgs, int32_t* out_ids, int32_t cap, int32_t* n_out);

OA_API const char* oa_last_error(void);                      /* thread-local message of the last failing call */
OA_API int oa_engine_stats(oa_engine*, char* buf, size_t n); /* JSON: steps, tokens, pages, launches, timings */
OA_API int oa_model_info(oa_engine*, char* buf, size_t n);   /* JSON: resolved architecture */

/* ---- native OpenAI-compatible HTTP front (csrc/http_server.cpp): what the UNMODIFIED reference binary is pointed at (`baseUrl` of POST /api/execute,
 * pkg/handlers/execute.go:21,205; OPENAI_API_BASE for the swarm flows, pkg/workflows/swarm.go:83).  POST /v1/chat/completions in go-openai's wire
 * format (openai.go:70-82) incl. `tools` -> grammar-forced `tool_calls`, GET /v1/models, GET /api/perf/stats.  One OS thread per connection; with
 * n_engines > 1 (data-parallel replicas, BASELINE configs[2]) conversations stick to the replica holding their prefix pages, new ones go to the
 * least-loaded replica, a replica over `max_inflight` answers 429 (openai.go:91-94 backs off).
 * options_json (flat): {"host":"127.0.0.1","port":0,"require_key":1,"api_key":"","tool_steps":3,"max_inflight":256,"max_connections":8192,"max_body_bytes":67108864,"idle_timeout_s":120} */
typedef struct oa_http oa_http;
OA_API int oa_http_start(oa_engine* const* engines, int32_t n_engines, const char* options_json, oa_http** out);
OA_API int32_t oa_http_port(oa_http*);                        /* the bound port (options "port": 0 picks a free one) */
OA_API int oa_http_stats(oa_http*, char* buf, size_t n);      /* JSON: requests, routed / in flight per replica, 429s, sticky hits, engine stats */
OA_API void oa_http_stop(oa_http*);                           /* stops accepting, waits for the connection threads; the engines stay alive */
OA_API const char* oa_http_last_error(void);

/* ---- measurement + parity hooks (used by bench.py and tests/; not part of the Go seam) ---- */
/* fresh single-sequence prefill of `tokens`; fp32 logits of every position -> logits_out[n, vocab] */
OA_API int oa_debug_prefill_logits(oa_engine*, const int32_t* tokens, int32_t n, float* logits_out);
/* Device-resident decode benchmark: builds `batch` sequences of `ctx_len` cached tokens (real chunked prefill of
 * seeded synthetic ids), then runs warmup+steps decode forwards of the whole batch, timed with CUDA events on the
 * engine stream.  out[0]=ms/step over ONE event bracket around all timed steps (host gaps included), out[1]=prefill ms, out[2]=kernel launches per step, out[3]=mean ctx over the
 * timed steps, out[4]=attention-kernel ms/step (avg), out[5]=algorithmic bytes/step,
 * out[6]=sum of per-step device durations / steps (host gaps excluded); with n_out >= 8 + batch, out[8 + b] = the token id sequence b
 * sampled in the last timed step; with n_out >= 8 + 2 * batch (single GPU), out[8 + batch + b] = that token's fp32 logit */
OA_API int oa_bench_decode(oa_engine*, int32_t batch, int32_t ctx_len, int32_t steps, int32_t warmup, double* out, int32_t n_out);
/* The same synthetic workload as oa_bench_decode (same tokens, pages and step inputs, no warmup steps, single GPU), untimed: the fp32
 * logits of every decode step -> logits_out[steps, batch, vocab] and the sampled ids -> ids_out[steps, batch].  mixed_rows > 0: the last
 * step also carries a mixed_rows-token prefill chunk of one extra sequence (a mixed step: decode attention for the batch, prefill
 * attention for the chunk); its row is not sampled. */
OA_API int oa_debug_decode_logits(oa_engine*, int32_t batch, int32_t ctx_len, int32_t steps, int32_t mixed_rows, float* logits_out, int32_t* ids_out);

/* in-situ per-kernel-class timings accumulated while OA_PROFILE_ALL=1 (JSON name -> [total ms, launches]) */
OA_API int oa_debug_kernel_times(oa_engine*, char* buf, size_t n, int32_t reset);

/* kernel-level entry points on raw device pointers (tests call these with torch-allocated memory) */
OA_API int oa_k_rmsnorm(const void* x, const void* gain, void* y, int32_t T, int32_t H, float eps, void* stream);
OA_API int oa_k_gemm(const void* A, const void* B, int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t block_n, void* out,
              const void* bias, const void* resid, float* logits, int32_t* argmax_out, void* stream);
/* persistent stream-K GEMM (M <= 128) followed by the fixed-order partial sum: out_f32[M,N] */
OA_API int oa_k_gemm_streamk(const void* A, const void* B, int32_t M, int32_t N, int32_t K, int32_t block_n, int32_t n_ctas, float* out_f32, void* stream);
OA_API int oa_k_init_weight(void* dst, uint64_t seed, uint64_t tensor_id, int64_t tensor_id_b, int64_t rows, int64_t cols, float std,
                     float mean, void* stream);
/* paged attention on a caller-provided cache [2(K,V)][num_pages][n_kv][64][D] (one layer): decode when q has one
 * row per sequence (n_q_rows == n_seqs), otherwise causal prefill of `q_lens[i]` new rows per sequence */
OA_API int oa_k_paged_attention(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables,
                         int32_t max_pages_per_seq, const int32_t* ctx_lens, const int32_t* q_lens, int32_t n_seqs,
                         int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t force_splits, void* stream);
/* the same on an fp8 (e4m3) cache of the same shape in bytes, each (page, kv head) block holding K as [64][D] and V transposed as [D][64];
 * K bytes decode to e4m3 * k_scale, V bytes to e4m3 * v_scale */
OA_API int oa_k_paged_attention_fp8(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables,
                             int32_t max_pages_per_seq, const int32_t* ctx_lens, const int32_t* q_lens, int32_t n_seqs,
                             int32_t n_heads, int32_t n_kv, int32_t head_dim, int32_t force_splits, float k_scale, float v_scale, void* stream);
/* the engine's RoPE + KV write (one layer) into such a cache: qkv [T, (n_heads + 2 n_kv) * D] bf16, positions / slots [T] and the RoPE
 * tables (fp32 [positions][D/2]) on the device; rotated q -> q_out [T, n_heads * D] */
OA_API int oa_k_kv_write_fp8(const void* qkv, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin,
                      void* q_out, void* kv_cache, int32_t num_pages, int32_t T, int32_t n_heads, int32_t n_kv, int32_t head_dim,
                      float k_scale, float v_scale, void* stream);
/* fp8 (e4m3) projections (weight_dtype "fp8_e4m3").  Row quantiser: bf16 x [R, C] -> e4m3 bytes q [R, C] + fp32 scale [R], per row
 * s = the smallest power of two with max|x| <= 448 s (all-zero row: 1), q = e4m3(x / s) (C % 16 == 0). */
OA_API int oa_k_quant_rows_e4m3(const void* x, void* q, float* scale, int32_t R, int32_t C, void* stream);
/* out = sa[m] * sb[n] * sum_k A[m,k] B[n,k] for e4m3 A [M, K], B [N, K] with fp32 row scales (device pointers); epilogues as oa_k_gemm
 * (0 store (+ bias), 1 residual, 2 SwiGLU), block_n in {32, 64, 128}; large shapes take the persistent kernel as in oa_k_gemm */
OA_API int oa_k_gemm_fp8(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t epilogue,
                         int32_t block_n, void* out, const void* bias, const void* resid, void* stream);
/* the same product on the stream-K decode GEMM (M <= 128, block_n 64 / 128): fuse 0 = fp32 out_f32 [M, N] (sum of the partials),
 * fuse 2 = x [M, N] bf16 += product, finished inside the GEMM */
OA_API int oa_k_gemm_streamk_fp8(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t block_n,
                                 int32_t n_ctas, int32_t fuse, void* x, float* out_f32, void* stream);
/* The decode step's finished projections, launched as DeviceModel::forward launches them (test entry points, not the serving path).  A [M, K]
 * and B [N, K] are bf16, or e4m3 bytes with fp32 row scales sa [M] / sb [N] (null for bf16).  path 0 = stream-K GEMM (block_n 64 / 128 / 256,
 * two 128-row slots when M > 128) + the stand-alone consumer; 1 = stream-K GEMM with the finisher fused (block_n 128); 2 / 3 / 4 / 8 = cluster
 * split-K with that cluster size (bf16).  Each call owns its stream-K workspace and zeroed tile flags.  A launcher's refusal returns
 * OA_ERR_BAD_REQUEST, any other CUDA error OA_ERR_INTERNAL. */
/* o / down: x [M, N] bf16 += A.B^T, then xn = rmsnorm(x) * gain; `launches` repeats both back to back on the same tile flags */
OA_API int oa_k_sk_row_parallel(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t N, int32_t K, int32_t block_n,
                                int32_t n_ctas, int32_t path, void* x, const void* gain, void* xn, float eps, int32_t launches, void* stream);
/* gate/up: act [M, F] = silu(gate) * up from B [2F, K] (16 gate rows, then 16 up rows per 32); paths 0 and 1 (bf16 only) */
OA_API int oa_k_sk_swiglu(const void* A, const float* sa, const void* B, const float* sb, int32_t M, int32_t F, int32_t K, int32_t block_n,
                          int32_t n_ctas, int32_t path, void* act, int32_t launches, void* stream);
/* qkv: (+ bias) -> bf16 -> RoPE -> q_out and one layer of a paged cache laid out as for oa_k_paged_attention (k_scale <= 0: bf16) or
 * oa_k_paged_attention_fp8; positions / slots [M] on the device */
OA_API int oa_k_sk_qkv_rope(const void* A, const float* sa, const void* B, const float* sb, const void* bias, int32_t M, int32_t K, int32_t n_heads,
                            int32_t n_kv, int32_t head_dim, int32_t block_n, int32_t n_ctas, int32_t path, const int32_t* positions, const int32_t* slots,
                            const float* rope_cos, const float* rope_sin, void* q_out, void* kv_cache, int32_t num_pages, float k_scale, float v_scale,
                            void* stream);
/* oa_k_kv_write_fp8 on a bf16 cache (the prefill writer) */
OA_API int oa_k_kv_write(const void* qkv, const int32_t* positions, const int32_t* slots, const float* rope_cos, const float* rope_sin, void* q_out,
                         void* kv_cache, int32_t num_pages, int32_t T, int32_t n_heads, int32_t n_kv, int32_t head_dim, void* stream);
/* decode attention on the engine's work plan for n_ctas_target CTAs (host block_tables / ctx_lens as oa_k_paged_attention).  merge_inline:
 * cut items are merged inside the kernel on merge counters zeroed once, `launches` times in a row; else by the separate merge kernel.
 * k_scale <= 0: bf16 cache */
OA_API int oa_k_decode_attention(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables,
                                 int32_t max_pages_per_seq, const int32_t* ctx_lens, int32_t n_seqs, int32_t n_heads, int32_t n_kv, int32_t head_dim,
                                 int32_t n_ctas_target, int32_t merge_inline, int32_t launches, float k_scale, float v_scale, void* stream);
/* the LM head: fp32 logits [M, N] and ids [M] = the arg-max of each row (ties: lowest id).  A row r with mask_slot[r] >= 0 takes it over the
 * ids whose bit (col_offset + column) is set in mask_table[mask_slot[r] * mask_words ...], 0 when none is (all device pointers) */
OA_API int oa_k_gemm_logits_masked(const void* A, const void* B, int32_t M, int32_t N, int32_t K, int32_t block_n, const uint32_t* mask_table,
                                   const int32_t* mask_slot, int32_t mask_words, int32_t col_offset, float* logits, int32_t* ids, void* stream);
/* The prefill step's tile-path kernels, launched as DeviceModel::forward launches them (test entry points, synchronous, each allocating what it
 * needs; a launcher's refusal returns OA_ERR_BAD_REQUEST).
 * Projection GEMM: A [a_rows, K] (a_rows >= M: the map spans a_rows rows, as the engine's activation maps span max_step_tokens) and B [N, K],
 * bf16, or e4m3 bytes with fp32 row scales sa / sb (null for bf16).  epilogue 0: out [M, N] = A.B^T (+ bias [N]); 1: out [M, N] += A.B^T in
 * place; 2: out [M, N/2] = silu(gate) * up (B rows 16 gate / 16 up per 32).  block_n 0 = the engine's choice (pick_bn, fp8 capped at 128);
 * the BLOCK_N used goes to *block_n_used.  The persistent or the tile kernel runs as launch_gemm decides (OA_GEMM_PERSISTENT /
 * OA_GEMM_PERSISTENT_MIN_TILES). */
OA_API int oa_k_prefill_gemm(const void* A, const float* sa, const void* B, const float* sb, int32_t a_rows, int32_t M, int32_t N, int32_t K,
                             int32_t epilogue, int32_t block_n, void* out, const void* bias, int32_t* block_n_used, void* stream);
/* One layer's attention of a prefill or mixed step on one paged cache (laid out as for oa_k_paged_attention, or oa_k_paged_attention_fp8 when
 * k_scale > 0).  Sequences 0 .. n_decode-1 have one query row each (rows 0 .. n_decode-1) and run decode attention on the engine's plan for
 * 2 x SMs CTAs with the in-kernel merge; the others have q_lens[i] rows each, the last at position ctx_lens[i] - 1, and run as the engine's
 * 128-row prefill tiles, heaviest first.  Both kernels on one stream, decode first.  block_tables / ctx_lens / q_lens on the host. */
OA_API int oa_k_step_attention(const void* q, void* out, const void* kv_cache, int32_t num_pages, const int32_t* block_tables,
                               int32_t max_pages_per_seq, const int32_t* ctx_lens, const int32_t* q_lens, int32_t n_seqs, int32_t n_decode,
                               int32_t n_heads, int32_t n_kv, int32_t head_dim, float k_scale, float v_scale, void* stream);
/* out [T, H] = table [vocab, H] rows of ids [T] (device); an id outside [0, vocab) reads row 0 */
OA_API int oa_k_embed_gather(const int32_t* ids, const void* table, void* out, int32_t T, int32_t H, int32_t vocab, void* stream);
/* The tensor-parallel collectives of DeviceModel::forward on one GPU (test entry points, synchronous).  Each collective reaches its peers through
 * a device table of pointers; here the t entries point at t local buffers, and ranks 0 .. t-1 run one after another on one stream, each with
 * the arguments that rank has on t GPUs.  Arrays of t device pointers are host arrays.  t outside 2..8 or a row length (H, K) that is not a
 * multiple of 8 returns OA_ERR_BAD_REQUEST, as does a launcher's refusal.
 * Decode o / down finish: per rank r, the stream-K GEMM of A[r] [M, K] by B[r] [H, K] (bf16; two 128-row slots when M > 128), its fp32 or
 * (bf16_partials) bf16 sum into partial[r] [M, H] with rank r's "buffer written" signal, then x[r] [M, H] += the rank-ordered sum of every
 * partial and xn[r] = rmsnorm(x[r]) * gain, after rank r's wait for the t signals.  flags: device uint32 [t][8] (rank p's flags are row p);
 * launch i uses epoch + i (wrapping).  The consumers of a launch run only once every one of the t x t flags shows its epoch, otherwise the
 * call returns OA_ERR_INTERNAL (oa_last_error names the flag).  `launches` repeats everything on the same flags and done counters. */
OA_API int oa_k_tp_row_parallel(int32_t t, const void* const* A, const void* const* B, int32_t M, int32_t H, int32_t K, int32_t block_n,
                                int32_t n_ctas, int32_t bf16_partials, void* const* partial, void* const* x, void* const* xn, const void* gain,
                                float eps, uint32_t* flags, uint32_t epoch, int32_t launches, void* stream);
/* Prefill all-reduce: x[r] [T, H] += the rank-ordered sum of the bf16 partials partial[·] [T, H], one-shot, or two-shot (rank r reduces
 * slice r of the flat T x H / 8 16-byte vectors into x[r] and gather[r], then copies every other rank's slice from gather[·]). */
OA_API int oa_k_tp_allreduce_prefill(int32_t t, void* const* partial, void* const* x, void* const* gather, int32_t T, int32_t H, int32_t two_shot,
                                     void* stream);
/* Vocab-parallel LM head: shard r = B rows [r V/t, (r+1) V/t) of B [V, K].  Its logits (optional: logits [M, V] at column r V/t), its
 * (max, lowest global id) per row into pairs[r] ({float, int32} [M]), then ids [M] = the best pair over the shards (ties: lowest id).
 * block_n 0 = the engine's choice for one shard.  A masked row (mask table as oa_k_gemm_logits_masked, bit = global id) with nothing
 * allowed gives (-inf, r V/t) on shard r and id 0.  V % t and (V / t) % 8 must be 0. */
OA_API int oa_k_tp_lm_head_argmax(int32_t t, const void* A, const void* B, int32_t M, int32_t V, int32_t K, int32_t block_n, const uint32_t* mask_table,
                                  const int32_t* mask_slot, int32_t mask_words, float* logits, void* const* pairs, int32_t* ids, void* stream);
/* ---- host-only logic, callable without a GPU (CPU tests) ---- */
/* BLOCK_N of the engine's tile-path GEMM [M, N] on sm_count SMs (pick_bn; override_bn in {32, 64, 128, 256} wins, fp8 != 0 caps it at 128) */
OA_API int32_t oa_host_pick_bn(int32_t M, int32_t N, int32_t sm_count, int32_t override_bn, int32_t fp8);
/* chat template + tokenizer of the model described by config_json */
OA_API int oa_host_apply_chat_template(const char* config_json, const oa_msg* msgs, int32_t n_msgs, int32_t* out_ids, int32_t cap, int32_t* n_out);
/* decode-attention work plan: segs_out[cap_segs*5] = {seq, kvh, chunk_begin, chunk_end, partial_slot}, cta_ptr_out[n_ctas+1];
 * returns the number of CTAs in *n_ctas_out and of segments in *n_segs_out */
OA_API int oa_host_decode_plan(const int32_t* ctx_lens, int32_t n_seqs, int32_t n_kv, int32_t n_ctas_target, int32_t force_splits,
                        int32_t* segs_out, int32_t cap_segs, int32_t* cta_ptr_out, int32_t cap_ctas, int32_t* n_ctas_out,
                        int32_t* n_segs_out, int32_t* n_slots_out);
/* stream-K unit plan of the decode projections (host only, no GPU): CTA c owns k-block units [cta_unit0[c], cta_unit0[c+1]) of
 * n_tiles x kb units (tile-major); tile_first/tile_last = the CTAs holding a tile's first and last k-block, computed with the
 * closed form the kernels use (floor(((u+1)*G-1)/total)).  The fused SwiGLU epilogue relies on: pieces of a tile are exactly
 * CTAs tile_first..tile_last, the first CTA's piece is the LAST segment of that CTA and every other piece is the FIRST segment
 * of its CTA (so the finishing CTA never waits on a CTA that is itself waiting). */
OA_API int oa_host_streamk_plan(int32_t N, int32_t K, int32_t block_n, int32_t n_ctas, int64_t* cta_unit0_out, int32_t cap_ctas,
                         int32_t* tile_first_out, int32_t* tile_last_out, int32_t cap_tiles, int32_t* n_ctas_out, int32_t* n_tiles_out,
                         int32_t* kb_out);
/* byte-level BPE tokenizer read from a Hugging Face tokenizer.json (Llama-3 / Qwen2.5 format), host only: what the engine uses
 * for text when its config names one ("tokenizer": path) instead of the synthetic byte-level vocabulary.  Loaded files are cached
 * by path.  encode: *n_out = number of ids (written up to cap; OA_ERR_BAD_REQUEST if cap is too small or the file is unsupported);
 * decode: bytes of the ids (control tokens render as their literal content). */
OA_API int oa_host_bpe_encode(const char* tokenizer_json_path, const char* text, int32_t text_len, int32_t* ids_out, int32_t cap, int32_t* n_out);
OA_API int oa_host_bpe_decode(const char* tokenizer_json_path, const int32_t* ids, int32_t n_ids, char* buf, int32_t cap, int32_t* n_out);
/* grammar automaton, host only: feeds `prefix` (n bytes) to the schema `kind` (1 tool call, 2 final) and returns the allowed-byte
 * bitset for the next position in mask_out[8], *done_out = 1 when the JSON is complete; 400 if the prefix is not derivable */
OA_API int oa_host_grammar_step(int32_t kind, const uint8_t* prefix, int32_t n, uint32_t* mask_out, int32_t* done_out);
OA_API int oa_host_grammar_step_ex(int32_t kind, const char* functions, const uint8_t* prefix, int32_t n, uint32_t* mask_out, int32_t* done_out);
/* token-level grammar mask, host only: the bitset (ceil(vocab/32) words) of token ids allowed after `prefix` under schema `kind`, for the
 * byte-level BPE vocabulary of tokenizer_json_path (NULL/"": the synthetic byte-level ids 0..255) — a token is allowed iff all of its bytes
 * walk the automaton.  key_out receives the canonical cache key of the state (states with equal keys have equal masks). */
OA_API int oa_host_grammar_token_mask(const char* tokenizer_json_path, int32_t vocab, int32_t kind, const char* functions, const uint8_t* prefix,
                               int32_t n, uint32_t* mask_out, int32_t cap_words, char* key_out, int32_t key_cap);
OA_API int oa_host_json_roundtrip(const uint8_t* in, size_t n_in, char* out, size_t n_out);   /* the HTTP front's JSON reader + writer, for the CPU tests */
/* resolved architecture + derived byte counts of a config, no device needed */
OA_API int oa_host_model_info(const char* config_json, char* buf, size_t n);
OA_API uint64_t oa_kernel_launches(void);
OA_API const char* oa_version(void);

#ifdef __cplusplus
}
#endif
#endif
