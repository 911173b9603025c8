"""Engine-level parity on the H100 (pytest -m gpu): the full decode path through the C ABI against the CPU
oracle in bf16-faithful mode on the same seeded weights and inputs (tiny configs that share every code path
with the 8B/32B/70B presets: GQA groups 2/4/5, head_dim 64/128, qkv bias, tied embeddings, llama3 rope scaling).

Stated tolerances (logits are O(1); see tests/test_oracle_golden.py::test_bf16_mode_close_to_fp32 for the bf16
noise floor of ~5e-2 between bf16-faithful and fp32 arithmetic):
    LOGIT_TOL  = 2.5e-2 absolute on fp32 logits, GPU vs oracle(bf16 mode)  — accumulation-order + exp2/expf effects
    token ids  : must be identical wherever the oracle's top1-top2 margin exceeds 2*LOGIT_TOL
"""
import dataclasses
import json
import os
import threading

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from opsagent_b200 import Engine, EngineError, LocalCUDAClient, ChatCompletionMessage, APIError  # noqa: E402
from oracle import oracle as O  # noqa: E402  (checker only)

LOGIT_TOL = 2.5e-2
CASES = ["tiny-llama", "tiny-llama-d128", "tiny-qwen"]


def make_engine(name, **kw):
    spec = O.PRESETS[name]
    cfg = spec.engine_json(num_pages=64, max_seq_len=512, max_batch=16, max_step_tokens=256)
    cfg.update(kw)
    return spec, Engine(cfg)


@pytest.fixture(scope="module", params=CASES)
def pair(request):
    spec, eng = make_engine(request.param)
    orc = O.Oracle(spec, max_pos=512, n_slots=1, mode=1)
    yield spec, eng, orc
    eng.close(); orc.close()


def test_prefill_logits_match_oracle(pair):
    spec, eng, orc = pair
    rng = np.random.default_rng(1)
    for n in (1, 17, 64, 65, 150, 256):        # <=128: stream-K one row tile; 129..256: two row tiles
        toks = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        got = eng.debug_prefill_logits(toks)
        ref = orc.forward(toks, all_logits=True)
        err = np.abs(got - ref).max()
        assert np.isfinite(got).all()
        assert err < LOGIT_TOL, (n, err)


def test_prefill_logits_through_persistent_gemm(monkeypatch):
    """same parity with every prefill projection forced through the persistent tile GEMM (the 8B prefill path)"""
    monkeypatch.setenv("OA_GEMM_PERSISTENT_MIN_TILES", "1")
    for name in CASES:
        spec, eng = make_engine(name, bn_qkv=128, bn_o=128, bn_gu=128, bn_down=128, max_step_tokens=512)
        orc = O.Oracle(spec, max_pos=512, mode=1)
        rng = np.random.default_rng(11)
        toks = rng.integers(0, spec.vocab, size=300).astype(np.int32)      # T > 256: tile-GEMM path, not stream-K
        got = eng.debug_prefill_logits(toks)
        ref = orc.forward(toks, all_logits=True)
        assert np.abs(got - ref).max() < LOGIT_TOL
        eng.close(); orc.close()


def test_two_row_tile_streamk_path_matches_oracle():
    """opt-in sk_max_rows=256: batches of 129..256 rows through the two-row-tile stream-K GEMM"""
    spec, eng = make_engine("tiny-llama-d128", sk_max_rows=256)
    orc = O.Oracle(spec, max_pos=512, mode=1)
    rng = np.random.default_rng(12)
    for n in (129, 200, 256):
        toks = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        assert np.abs(eng.debug_prefill_logits(toks) - orc.forward(toks, all_logits=True)).max() < LOGIT_TOL
    eng.close(); orc.close()


@pytest.mark.parametrize("name", CASES + ["llama-3.2-1b"])
def test_fused_decode_epilogues_are_bit_identical_to_separate_kernels(name):
    """Baseline: one kernel per projection and per consumer (sk_fuse_swiglu=0, sk_fuse_epi=0).  Variants: the qkv projection
    finishing bias + RoPE + the paged-KV write and the o / down projections finishing the residual add in their own epilogues
    (sk_fuse_epi bitmask 1 / 2 / 4; o and down are followed by a norm-only kernel with the consumer's reduction order); the gate/up projection finishing
    SwiGLU in its own epilogue (the CTA holding a tile's first k-block adds the other CTAs' pieces in CTA order).  Reduction order and consumer code are shared, so logits and generated ids must be EQUAL, not close.
    llama-3.2-1b exercises real multi-CTA tile splits on all 132 SMs."""
    full = name == "llama-3.2-1b"
    rng = np.random.default_rng(77)
    spec = O.PRESETS[name]
    prompts = [rng.integers(0, spec.vocab if not full else 256, size=n).astype(np.int32) for n in ((1, 33, 128) if not full else (7, 128))]
    gen_prompts = [rng.integers(0, 256, size=n).astype(np.int32).tolist() for n in (3, 19, 40, 64, 90)]
    variants = [dict(sk_fuse_swiglu=0, sk_fuse_epi=0), dict(sk_fuse_swiglu=1, sk_fuse_epi=0), dict(sk_fuse_swiglu=0, sk_fuse_epi=7),
                dict(sk_fuse_swiglu=1, sk_fuse_epi=1), dict(sk_fuse_swiglu=1, sk_fuse_epi=6)]
    results = []
    for kw in variants:
        if full:
            eng = Engine({"model": name, "num_pages": 64, "max_seq_len": 512, "max_batch": 8, "max_step_tokens": 512, "seed": spec.seed, **kw})
        else:
            _, eng = make_engine(name, **kw)
        logits = [eng.debug_prefill_logits(t) for t in prompts]
        # one request at a time keeps the batch composition (and with it the attention work plan) identical across variants;
        # twice: the tile flags must re-arm between launches
        outs = []
        for _ in range(2):
            outs.append([list(eng.generate(pt, 12 if full else 30, flags=1).token_ids) for pt in gen_prompts])
        results.append((logits, outs))
        eng.close()
    for kw, res in zip(variants[1:], results[1:]):
        for a, b in zip(results[0][0], res[0]):
            assert np.array_equal(a, b), f"{kw}: logits differ by {np.abs(a - b).max()}"
        assert results[0][1] == res[1], f"{kw}: generated ids differ"
    assert results[0][1][0] == results[0][1][1]


def test_long_context_chunked_prefill_and_decode_match_oracle():
    """5000-token prompt prefilled in 2048-token chunks over several scheduler steps (each chunk attends to the cached pages of
    the earlier ones), then decode over ~80 pages with split/merged attention segments — llama3 RoPE scaling, head_dim 128."""
    spec, eng = make_engine("tiny-llama-d128", max_seq_len=8192, num_pages=200, max_step_tokens=2048, max_batch=4)
    orc = O.Oracle(spec, max_pos=5200, mode=1)
    rng = np.random.default_rng(31)
    prompt = rng.integers(0, spec.vocab, size=5000).astype(np.int32)
    ref, margins, _ = orc.generate(prompt, 12)
    out = eng.generate(prompt.tolist(), 12, flags=1)
    k = 0
    while k < 12 and ref[k] == out.token_ids[k]:
        k += 1
    assert k == 12 or margins[k] <= 2 * LOGIT_TOL, (k, margins[k])
    st = eng.stats()
    assert st["prefill_steps"] >= 3 and st["prefill_tokens"] == 5000
    eng.close(); orc.close()


def test_greedy_generation_matches_oracle(pair):
    spec, eng, orc = pair
    rng = np.random.default_rng(2)
    for n, g in ((5, 40), (70, 24), (130, 70)):
        prompt = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        ref, margins, _ = orc.generate(prompt, g)
        out = eng.generate(prompt.tolist(), g, flags=1)
        assert out.completion_tokens == g and out.finish_reason == "length"
        for i, (a, b) in enumerate(zip(out.token_ids, ref)):
            if a != b:
                assert margins[i] <= 2 * LOGIT_TOL, f"token {i}: engine {a} oracle {b} margin {margins[i]}"
                break          # after a legitimate near-tie flip the continuations differ
        else:
            assert list(out.token_ids) == list(ref)


def test_chat_template_and_content_match_oracle(pair):
    spec, eng, orc = pair
    msgs = [("system", "You are a Kubernetes expert. 你是一名K8s专家"), ("user", "how many namespace in the cluster?")]
    ids = eng.apply_chat_template(msgs)
    assert ids == O.apply_chat_template(spec, msgs)
    assert eng.count_tokens(msgs) == len(ids)
    ref, margins, _ = orc.generate(np.array(ids, np.int32), 16, eos=O.eos_ids(spec))
    out = eng.chat_complete(spec.name, msgs, 16)
    k = 0
    while k < min(len(ref), len(out.token_ids)) and ref[k] == out.token_ids[k]:
        k += 1
    if k < min(len(ref), len(out.token_ids)):
        assert margins[k] <= 2 * LOGIT_TOL
    else:
        assert out.content == O.detokenize(ref)
    assert out.prompt_tokens == len(ids)


def test_concurrent_requests_equal_sequential():
    """Many goroutine-style blocking callers batched into shared forwards must each get what they would get alone
    (continuous batching, chunked prefill and ragged paged decode do not change results beyond near-ties)."""
    spec, eng = make_engine("tiny-llama", max_step_tokens=128)
    orc = O.Oracle(spec, max_pos=512, mode=1)
    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, spec.vocab, size=int(n)).astype(np.int32) for n in rng.integers(3, 200, size=24)]
    gens = [int(g) for g in rng.integers(4, 40, size=24)]
    results = [None] * len(prompts)

    def worker(i):
        results[i] = eng.generate(prompts[i].tolist(), gens[i], flags=1)

    th = [threading.Thread(target=worker, args=(i,)) for i in range(len(prompts))]
    [t.start() for t in th]; [t.join() for t in th]
    n_exact = 0
    for i, r in enumerate(results):
        ref, margins, _ = orc.generate(prompts[i], gens[i])
        assert r.completion_tokens == gens[i]
        k = 0
        while k < gens[i] and ref[k] == r.token_ids[k]:
            k += 1
        if k == gens[i]:
            n_exact += 1
        else:
            assert margins[k] <= 2 * LOGIT_TOL, (i, k, margins[k])
    assert n_exact >= len(prompts) // 2
    st = eng.stats()
    assert st["requests_completed"] == len(prompts) and st["pages_free"] == st["pages_total"]
    assert st["decode_steps"] < sum(gens)          # really batched
    eng.close(); orc.close()


def test_preemption_and_page_recycling():
    """A KV pool too small for all requests at once: sequences are preempted (recompute) and still finish right."""
    spec, eng = make_engine("tiny-llama", num_pages=8, max_seq_len=256, max_batch=8)
    orc = O.Oracle(spec, max_pos=256, mode=1)
    rng = np.random.default_rng(4)
    prompts = [rng.integers(0, spec.vocab, size=60).astype(np.int32) for _ in range(6)]
    tickets = [eng.tokens_submit(p.tolist(), 100, flags=1) for p in prompts]
    outs = [eng.wait(t) for t in tickets]
    for p, o in zip(prompts, outs):
        ref, margins, _ = orc.generate(p, 100)
        k = 0
        while k < 100 and ref[k] == o.token_ids[k]:
            k += 1
        assert k == 100 or margins[k] <= 2 * LOGIT_TOL
    st = eng.stats()
    assert st["preemptions"] > 0 and st["pages_free"] == st["pages_total"]
    eng.close(); orc.close()


def test_error_codes_follow_the_reference_contract():
    spec, eng = make_engine("tiny-llama", max_seq_len=128)
    with pytest.raises(EngineError) as e:
        eng.chat_complete("gpt-4", [("user", "hi")], 8)          # unknown model -> 400, fails fast (openai.go:96)
    assert e.value.code == 400
    with pytest.raises(EngineError) as e:
        eng.generate(list(range(200)), 8)                        # prompt longer than the KV budget -> 400
    assert e.value.code == 400
    with pytest.raises(EngineError) as e:
        eng.chat_complete(spec.name, [], 8)                       # "prompts cannot be empty" (simple.go:312)
    assert e.value.code == 400
    # the Go-mirror client maps codes to APIError and returns content as str
    cli = LocalCUDAClient(eng, sleep=lambda s: None)
    txt = cli.Chat(spec.name, 6, [ChatCompletionMessage("user", "hello")])
    assert isinstance(txt, str)
    with pytest.raises(APIError):
        cli.Chat("nope", 6, [ChatCompletionMessage("user", "hello")])
    eng.close()


def test_eos_stops_generation():
    """With EOS honoured the engine stops exactly where the oracle does."""
    spec, eng = make_engine("tiny-qwen")
    orc = O.Oracle(spec, max_pos=512, mode=1)
    rng = np.random.default_rng(6)
    # random-init logits rarely pick EOS; declare the oracle's own 5th token the stop id by checking prefix behaviour
    prompt = rng.integers(0, spec.vocab, size=20).astype(np.int32)
    ref, margins, _ = orc.generate(prompt, 12)
    out = eng.generate(prompt.tolist(), 12)
    assert out.finish_reason in ("length", "stop")
    assert out.completion_tokens <= 12
    eng.close(); orc.close()


@pytest.mark.parametrize("kind,flag", [(O.GRAMMAR_TOOLCALL, 2), (O.GRAMMAR_FINAL, 4)])
def test_grammar_constrained_completion_is_toolprompt_json_and_matches_oracle(kind, flag):
    """OA_FLAG_JSON_*: the completion parses as tools.ToolPrompt (reference pkg/tools/tool.go:29-38) and equals the oracle's
    constrained greedy decode on the same weights wherever the margin among the allowed bytes exceeds the tolerance."""
    import json as _json
    spec, eng = make_engine("tiny-llama", max_seq_len=1024, num_pages=64)
    orc = O.Oracle(spec, max_pos=1024, mode=1)
    msgs = [("system", "You are a Kubernetes expert."), ("user", "how many namespace in the cluster?")]
    ids = eng.apply_chat_template(msgs)
    out = eng.chat_complete(spec.name, msgs, 700, flags=flag)
    doc = _json.loads(out.content.decode("ascii"))
    assert list(doc.keys()) == ["question", "thought", "action", "observation", "final_answer"] and out.finish_reason == "stop"
    if kind == O.GRAMMAR_TOOLCALL:
        assert doc["action"]["name"] in O.TOOLS and doc["final_answer"] == ""
    else:
        assert len(doc["final_answer"]) >= 10
    ref, margins, _ = O.generate_constrained(orc, np.array(ids, np.int32), kind)
    got = out.content
    k = 0
    while k < min(len(ref), len(got)) and ref[k] == got[k]:
        k += 1
    assert k == len(ref) == len(got) or margins[k] <= 2 * LOGIT_TOL, (k, margins[k] if k < len(margins) else None)
    eng.close(); orc.close()


def test_json_mode_drives_a_multi_step_react_loop():
    """engine option json_mode: tool-call steps first, then a final answer, decided from the resent history
    (reference pkg/assistants/simple.go:391-501) — mixed with unconstrained requests in the same batch."""
    import json as _json
    spec, eng = make_engine("tiny-llama", max_seq_len=4096, num_pages=160, json_mode=1, react_tool_steps=2)
    history = [("system", "sys"), ("user", "why is pod web-0 crashing?")]
    names = []
    for step in range(3):
        raw = eng.generate(list(range(50, 90)), 8, flags=1)            # an unconstrained request keeps running alongside
        assert raw.completion_tokens == 8
        out = eng.chat_complete(spec.name, history, 700)
        doc = _json.loads(out.content.decode("ascii"))
        if step < 2:
            assert doc["action"]["name"] in O.TOOLS and doc["final_answer"] == ""
            names.append(doc["action"]["name"])
            doc["observation"] = "NAME READY STATUS\nweb-0 0/1 CrashLoopBackOff"
            history += [("assistant", out.content.decode("ascii")), ("user", _json.dumps(doc))]
        else:
            assert doc["action"]["name"] == "" and len(doc["final_answer"]) >= 10
    eng.close()


def test_prefix_cache_reuses_history_pages_without_changing_results():
    """step k of a ReAct conversation resends step k-1's prompt + reply + observation (reference simple.go:498-501): the shared
    prefix must come from cached KV pages, results must stay oracle-exact, and the pool must drain back to empty."""
    spec, eng = make_engine("tiny-llama", max_seq_len=1024, num_pages=48, max_batch=8)
    orc = O.Oracle(spec, max_pos=1024, mode=1)
    rng = np.random.default_rng(21)
    base = rng.integers(0, spec.vocab, size=300).astype(np.int32)
    r1 = eng.generate(base.tolist(), 20, flags=1)
    s1 = eng.stats()
    assert s1["prefix_hit_tokens"] == 0 and s1["pages_cached"] >= 4
    # same prompt again: everything but the last partial page comes from the cache, same tokens out
    r2 = eng.generate(base.tolist(), 20, flags=1)
    s2 = eng.stats()
    assert s2["prefix_hit_tokens"] == 256 and list(r2.token_ids) == list(r1.token_ids)
    assert s2["prefill_tokens"] - s1["prefill_tokens"] == 300 - 256
    # next "ReAct step": previous prompt + reply + new observation
    nxt = np.concatenate([base, np.array(r1.token_ids, np.int32), rng.integers(0, spec.vocab, size=90).astype(np.int32)])
    r3 = eng.generate(nxt.tolist(), 16, flags=1)
    s3 = eng.stats()
    # 4 full pages: the KV of the last generated token (index 319) is never computed, so page 4 (tokens 256..319) stayed incomplete
    assert s3["prefix_hit_tokens"] - s2["prefix_hit_tokens"] == 256
    ref, margins, _ = orc.generate(nxt, 16)
    k = 0
    while k < 16 and ref[k] == r3.token_ids[k]:
        k += 1
    assert k == 16 or margins[k] <= 2 * LOGIT_TOL
    # a different prefix does not hit; concurrent identical prompts are all correct
    other = rng.integers(0, spec.vocab, size=200).astype(np.int32)
    tickets = [eng.tokens_submit(other.tolist(), 10, flags=1) for _ in range(6)]
    outs = [eng.wait(t) for t in tickets]
    assert all(list(o.token_ids) == list(outs[0].token_ids) for o in outs)
    # eviction: fill the pool with new prefixes, everything still completes and all references are dropped
    for i in range(12):
        eng.generate(rng.integers(0, spec.vocab, size=400).astype(np.int32).tolist(), 4, flags=1)
    st = eng.stats()
    assert st["pages_free"] == st["pages_total"] and st["pages_cached"] <= st["pages_total"]
    eng.close(); orc.close()


# ---- full-size parity: the models BASELINE.json names, same seeded weights on both sides --------------------------------------
def _bpe_template_ids(tokenizer_json, msgs):
    """llama3 chat template over a byte-level BPE, built with the Hugging Face `tokenizers` library itself (independent of csrc/bpe.hpp)"""
    tokenizers = pytest.importorskip("tokenizers")
    t = tokenizers.Tokenizer.from_file(tokenizer_json)
    sp = {n: t.token_to_id(n) for n in ("<|begin_of_text|>", "<|start_header_id|>", "<|end_header_id|>", "<|eot_id|>")}
    enc = lambda s: t.encode(s, add_special_tokens=False).ids      # noqa: E731
    ids = [sp["<|begin_of_text|>"]]
    for role, content in msgs:
        ids += [sp["<|start_header_id|>"]] + enc(role) + [sp["<|end_header_id|>"]] + enc("\n\n") + enc(content) + [sp["<|eot_id|>"]]
    return ids + [sp["<|start_header_id|>"]] + enc("assistant") + [sp["<|end_header_id|>"]] + enc("\n\n")


def _full_size_parity(name, prompt, n_new, kv_pages, tokenizer=None, logit_rows=None, floor=None, overrides=None):
    """At 16-80 layers the bf16 rounding of every stored activation makes two bf16 computations with different fp32 accumulation
    orders drift apart chaotically: the CPU oracle in bf16-faithful mode itself sits `floor` away from its own fp32 mode.  Stated
    tolerance at full size: the engine's fp32 logits must be as close to the oracle's fp32-activation logits as 1.5x that floor
    (max and mean), and greedy tokens must agree wherever the oracle's top-1 margin exceeds 2x the floor.
    tokenizer: a tokenizer.json (the prompt is then the reference's real text through a real BPE); logit_rows: prompt positions whose
    logits are compared (default: all).  floor = (max, mean) measured by an earlier call on the same model: the fp32-mode oracle pass is
    then skipped (a 1,536-token prompt costs minutes of CPU per pass) and the engine is compared with the bf16-faithful oracle directly,
    within 2.5x the floor (triangle inequality: 1.5x to the fp32 oracle + 1x between the oracle's two modes).
    prompt: chat messages [(role, content)] (through the chat template) or the prompt's token ids.  overrides: preset fields replaced on both
    sides (engine config and ModelSpec), e.g. fewer layers and random norm gains."""
    overrides = overrides or {}
    spec = dataclasses.replace(O.PRESETS[name], **overrides)
    cfg = {"model": name, "num_pages": kv_pages, "max_seq_len": 2048, "max_batch": 8, "max_step_tokens": 2048, "seed": spec.seed, **overrides}
    if tokenizer:
        cfg["tokenizer"] = tokenizer
    eng = Engine(cfg)
    chat = isinstance(prompt[0], tuple)
    if chat:
        ids = eng.apply_chat_template(prompt)
        assert ids == (_bpe_template_ids(tokenizer, prompt) if tokenizer else O.apply_chat_template(spec, prompt))
    else:
        ids = [int(t) for t in prompt]
    toks = np.array(ids, np.int32)
    rows = list(range(len(ids))) if logit_rows is None else [r if r >= 0 else len(ids) + r for r in logit_rows]
    got = eng.debug_prefill_logits(ids)[rows]
    out = eng.chat_complete(name, prompt, n_new, flags=1) if chat else eng.generate(ids, n_new, flags=1)
    eng.close()
    assert np.isfinite(got).all()
    orc1 = O.Oracle(spec, max_pos=len(ids) + n_new + 8, mode=1)
    ref1_all = orc1.forward(toks, all_logits=True)
    ref1, ref1_last = ref1_all[rows], ref1_all[-1].copy()
    del ref1_all
    if floor is None:
        orc0 = O.Oracle(spec, max_pos=len(ids) + n_new + 8, mode=0)
        ref0 = orc0.forward(toks, all_logits=True)[rows]
        orc0.close()
        floor_max, floor_mean = float(np.abs(ref1 - ref0).max()), float(np.abs(ref1 - ref0).mean())
        err_max, err_mean = float(np.abs(got - ref0).max()), float(np.abs(got - ref0).mean())
        assert err_max <= 1.5 * floor_max + 1e-3 and err_mean <= 1.5 * floor_mean + 1e-4, (err_max, floor_max, err_mean, floor_mean)
    else:
        floor_max, floor_mean = floor
        err_max, err_mean = float(np.abs(got - ref1).max()), float(np.abs(got - ref1).mean())
        assert err_max <= 2.5 * floor_max + 1e-3 and err_mean <= 2.5 * floor_mean + 1e-4, (err_max, floor_max, err_mean, floor_mean)
    # greedy continuation from the KV state the prefill above left in the oracle (no second prefill of a long prompt)
    ref_t, margins = [], []
    lg = ref1_last
    for i in range(n_new):
        order = np.argsort(lg)
        ref_t.append(int(order[-1]) if lg[order[-1]] > lg[order[-2]] else int(min(order[-1], order[-2])))
        margins.append(float(abs(lg[order[-1]] - lg[order[-2]])))
        if i + 1 < n_new:
            lg = orc1.forward(np.array([ref_t[-1]], np.int32), pos0=len(ids) + i)[0]
    orc1.close()
    k = 0
    while k < n_new and out.token_ids[k] == ref_t[k]:
        k += 1
    assert k == n_new or margins[k] <= 2 * floor_max, (k, margins[k], floor_max)
    return {"prompt_tokens": len(ids), "err_max": err_max, "err_mean": err_mean, "floor_max": floor_max, "floor_mean": floor_mean, "same_tokens": k}


K8S_BPE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bpe_k8s_8k.json")


def test_full_size_llama_3_2_1b_execute_prompt_matches_oracle():
    """BASELINE configs[0]: the single `execute` question of the reference's README (README.md:247) exactly as POST /api/execute builds it
    (pkg/handlers/execute.go:190-199: system = executeSystemPrompt_cn VERBATIM, user = the cleaned instructions) on Llama-3.2-1B (tied
    embeddings, llama3 RoPE scaling, head_dim 64), tokenised by a real byte-level BPE; logits of every prompt position and 32 greedy tokens."""
    from opsagent_b200 import workloads as WL
    msgs = [(m.Role, m.Content) for m in WL.execute_messages("execute how many namespace in the cluster?")]
    assert msgs[0][1] == WL.prompt("executeSystemPrompt_cn") and len(msgs[0][1].encode()) == 3233
    print("llama-3.2-1b:", _full_size_parity("llama-3.2-1b", msgs, 32, 64, tokenizer=K8S_BPE))


def test_full_size_llama_3_8b_matches_oracle():
    """the bench model itself (BASELINE configs[1]) on the bench's own request: the analyze flow's verbatim prompt + a synthetic Pod
    manifest padded to P = 1536 tokens; fp32 logits at early, middle and the last prompt positions (RoPE phase and pages past position
    1,500) and 32 greedy tokens vs the CPU oracle.  Short prompt first (every position), as in round 1."""
    from opsagent_b200 import workloads as WL
    msgs = [("user", "why is pod web-0 in CrashLoopBackOff?")]
    short = _full_size_parity("llama-3-8b", msgs, 6, 64)
    print("llama-3-8b short:", short)
    if os.environ.get("OA_SKIP_SLOW_PARITY"):      # dev iteration only: the long-prompt half costs minutes of CPU oracle time
        return
    P = 1536 if (os.cpu_count() or 1) >= 16 else 640      # one bf16-faithful CPU oracle pass: ~3 minutes for 1,536 tokens on 16 cores
    tmp = Engine({"model": "tiny-llama", "hidden": 256, "n_layers": 1, "n_heads": 4, "n_kv_heads": 2, "head_dim": 64, "ffn": 256, "vocab": 8192,
                  "num_pages": 40, "max_seq_len": 2048, "tokenizer": K8S_BPE})             # only its tokenizer is used, to fit the manifest
    m = WL.fit_to_tokens(WL.analyze_messages, WL.synthetic_pod_yaml(7, 12 * P), P, tmp.count_tokens)
    tmp.close()
    msgs = [(x.Role, x.Content) for x in m]
    res = _full_size_parity("llama-3-8b", msgs, 32, 64, tokenizer=K8S_BPE, logit_rows=[0, 5, 300, P // 2, -130, -64, -3, -2, -1],
                            floor=(short["floor_max"], short["floor_mean"]))
    assert res["prompt_tokens"] == P
    print("llama-3-8b analyze:", res)


@pytest.mark.parametrize("name", ["llama-3-8b", "qwen2.5-32b", "llama-3-70b"])
def test_production_width_with_random_norm_gains_matches_oracle(name):
    """The production widths through DeviceModel::forward on one GPU, two layers deep: Llama-3-8B, Qwen2.5-32B (qkv bias at H = 5120,
    rope theta 1e6, eps 1e-6, untied 152,064-row head) and Llama-3-70B (H = 8192, 64 query heads).  Random norm gains (the presets have
    gains of exactly 1): a gain applied in the wrong place — ln2 for ln1, the next layer's ln1 for the final norm — changes the logits.
    Prompts of 1 and 37 tokens (one stream-K row tile), 128 (a full one) and 200 (the tile path); logits of every prompt row and 12 greedy
    tokens, within the full-size floor rule of _full_size_parity."""
    spec = O.PRESETS[name]
    rng = np.random.default_rng(42)
    for n in (1, 37, 128, 200):
        toks = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        res = _full_size_parity(name, toks, 12, 64, overrides=dict(n_layers=2, norm_random=1))
        print(f"{name} n_layers=2 norm_random=1 prompt {n}:", res)


@pytest.mark.parametrize("front", ["native", "python"])
def test_http_front_function_calling_end_to_end_matches_oracle(front):
    """the swarm-go wire path (reference pkg/workflows/swarm.go:14-78, analyze.go:47-75): POST /v1/chat/completions with `tools`
    -> grammar-forced tool_calls whose bytes equal the oracle's constrained greedy decode; then a text answer."""
    import json as _json
    import urllib.request
    from opsagent_b200.http_front import serve
    spec, eng = make_engine("tiny-llama", max_seq_len=2048, num_pages=96)
    orc = O.Oracle(spec, max_pos=1024, mode=1)
    if front == "native":
        from opsagent_b200.native_front import NativeFront
        srv = NativeFront([eng], tool_steps=1)
        port = srv.port
    else:
        srv, _ = serve(eng, port=0, tool_steps=1)
        port = srv.server_address[1]
    url = f"http://127.0.0.1:{port}/v1/chat/completions"
    tools = [{"type": "function", "function": {"name": "kubectl", "parameters": {"type": "object", "properties": {"command": {"type": "string"}}}}},
             {"type": "function", "function": {"name": "trivy", "parameters": {"type": "object", "properties": {"image": {"type": "string"}}}}}]
    msgs = [{"role": "system", "content": "You are an expert Kubernetes analyst."}, {"role": "user", "content": "analyze pod web-0"}]

    def post(body):
        rq = urllib.request.Request(url, data=_json.dumps(body).encode(), headers={"Content-Type": "application/json", "Authorization": "Bearer sk-local"})
        return _json.loads(urllib.request.urlopen(rq, timeout=120).read())

    r = post({"model": spec.name, "messages": msgs, "tools": tools, "max_tokens": 400, "temperature": 1.4e-45})
    tc = r["choices"][0]["message"]["tool_calls"][0]
    assert r["choices"][0]["finish_reason"] == "tool_calls" and tc["function"]["name"] in ("kubectl", "trivy")
    args = _json.loads(tc["function"]["arguments"])
    assert list(args.keys()) == [{"kubectl": "command", "trivy": "image"}[tc["function"]["name"]]]
    ids = O.apply_chat_template(spec, [(m["role"], m["content"]) for m in msgs])
    ref, margins, _ = O.generate_constrained(orc, np.array(ids, np.int32), O.GRAMMAR_FUNCTION, functions="kubectl:command,trivy:image")
    got = ('{"name":"%s","arguments":{"%s":"%s"}}' % (tc["function"]["name"], list(args.keys())[0], list(args.values())[0])).encode()
    k = 0
    while k < min(len(ref), len(got)) and ref[k] == got[k]:
        k += 1
    assert k == len(ref) == len(got) or margins[k] <= 2 * LOGIT_TOL
    msgs2 = msgs + [{"role": "assistant", "tool_calls": [tc]}, {"role": "tool", "tool_call_id": tc["id"], "content": "web-0 0/1 CrashLoopBackOff"}]
    r2 = post({"model": spec.name, "messages": msgs2, "tools": tools, "max_tokens": 400})
    assert r2["choices"][0]["finish_reason"] == "stop" and 10 <= len(r2["choices"][0]["message"]["content"]) <= 200
    srv.shutdown(); eng.close(); orc.close()


@pytest.mark.parametrize("name,dtype", [("tiny-llama", "BF16"), ("tiny-qwen", "F32"), ("tiny-llama-d128", "BF16")])
def test_safetensors_checkpoint_loading(name, dtype, tmp_path):
    """weights from a Hugging Face style checkpoint (HF tensor names, fused q|k|v, interleaved gate/up, tied / untied head,
    qkv bias, fp32 -> bf16 conversion): the engine is created with a DIFFERENT seed, so only a correct load reproduces the oracle."""
    spec = O.PRESETS[name]
    orc = O.Oracle(spec, max_pos=512, mode=1)
    path = str(tmp_path / "model.safetensors")
    O.write_safetensors(orc, path, dtype)
    cfg = spec.engine_json(num_pages=32, max_seq_len=512, max_batch=4, max_step_tokens=256, weights=path)
    cfg["seed"] = 987654321
    eng = Engine(cfg)
    rng = np.random.default_rng(17)
    for n in (9, 150):
        toks = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        assert np.abs(eng.debug_prefill_logits(toks) - orc.forward(toks, all_logits=True)).max() < LOGIT_TOL
    eng.close(); orc.close()
    with pytest.raises(EngineError):
        Engine(spec.engine_json(num_pages=32, max_seq_len=512, weights=str(tmp_path / "missing.safetensors")))


def test_malformed_checkpoints_are_refused_with_a_message(tmp_path):
    """wrong-config, transposed and truncated checkpoints must fail engine creation cleanly (no out-of-bounds read of the mapping)"""
    import struct
    spec = O.PRESETS["tiny-llama"]
    orc = O.Oracle(spec, max_pos=64, mode=1)
    good = str(tmp_path / "good.safetensors")
    O.write_safetensors(orc, good, "BF16")
    orc.close()
    raw = open(good, "rb").read()
    hl = struct.unpack("<Q", raw[:8])[0]
    header = json.loads(raw[8:8 + hl])

    def write(path, hdr, body):
        hj = json.dumps(hdr, separators=(",", ":")).encode()
        hj += b" " * ((8 - len(hj) % 8) % 8)
        open(path, "wb").write(struct.pack("<Q", len(hj)) + hj + body)

    # (1) a checkpoint of another architecture: engine configured with twice the ffn
    cfg = spec.engine_json(num_pages=32, max_seq_len=512, weights=good)
    cfg["ffn"] = spec.ffn * 2
    with pytest.raises(EngineError, match="shape"):
        Engine(cfg)
    # (2) same element count, transposed shape
    h2 = json.loads(json.dumps(header))
    k = "model.layers.0.mlp.down_proj.weight"
    h2[k]["shape"] = h2[k]["shape"][::-1]
    p2 = str(tmp_path / "transposed.safetensors"); write(p2, h2, raw[8 + hl:])
    with pytest.raises(EngineError, match="shape"):
        Engine(spec.engine_json(num_pages=32, max_seq_len=512, weights=p2))
    # (3) data_offsets that do not cover prod(shape) * sizeof(dtype)
    h3 = json.loads(json.dumps(header))
    k = "model.layers.0.mlp.gate_proj.weight"
    h3[k]["data_offsets"][1] -= 64
    p3 = str(tmp_path / "short.safetensors"); write(p3, h3, raw[8 + hl:])
    with pytest.raises(EngineError, match="data_offsets"):
        Engine(spec.engine_json(num_pages=32, max_seq_len=512, weights=p3))
    # (4) file cut in the middle of the tensor data
    p4 = str(tmp_path / "cut.safetensors"); open(p4, "wb").write(raw[: len(raw) // 2])
    with pytest.raises(EngineError):
        Engine(spec.engine_json(num_pages=32, max_seq_len=512, weights=p4))


def test_cancel_model_aliases_and_oversize_text():
    """oa_chat_cancel frees an abandoned request's pages (a timed-out wait would otherwise decode to max_tokens), `model_aliases`
    lets the engine answer to the names the unmodified reference sends (execute.go:168-171: currentModel or "gpt-4"), and text that
    cannot possibly fit is refused before it is tokenised"""
    import time
    spec, eng = make_engine("tiny-llama", model_aliases="gpt-4,gpt-4o")
    assert eng.chat_complete("gpt-4", [("user", "hi")], 4, flags=1).completion_tokens == 4
    with pytest.raises(EngineError) as e:
        eng.chat_complete("claude", [("user", "hi")], 4)
    assert e.value.code == 400 and "model_aliases" in e.value.message
    with pytest.raises(EngineError) as e:
        eng.chat_complete(spec.name, [("user", "x" * (512 * 16 + 1))], 4)
    assert e.value.code == 400 and "cannot fit" in e.value.message
    # a long request is decoding; the caller gives up
    t = eng.tokens_submit(list(range(1, 40)), 400, flags=1)
    with pytest.raises(EngineError) as e:
        eng.wait(t, timeout_ms=1)
    assert e.value.code == 408
    eng.cancel(t)
    with pytest.raises(EngineError):
        eng.wait(t, timeout_ms=1)                                   # the ticket is gone
    t_end = time.time() + 10
    while time.time() < t_end:
        st = eng.stats()
        if st["running"] == 0 and st["pages_free"] + st["pages_cached"] == st["pages_total"]:
            break
        time.sleep(0.005)
    st = eng.stats()
    assert st["cancelled"] == 1 and st["running"] == 0 and st["pages_free"] + st["pages_cached"] == st["pages_total"]
    # a cancelled WAITING request (engine busy elsewhere) and normal service afterwards
    out = eng.generate([5, 6, 7], 8, flags=1)
    assert out.completion_tokens == 8
    eng.close()
    spec, eng = make_engine("tiny-llama", model_aliases="*")
    assert eng.chat_complete("whatever-the-caller-says", [("user", "hi")], 3, flags=1).completion_tokens == 3
    eng.close()


def test_benchmarked_batch_geometry_matches_oracle():
    """What bench.py TIMES is a decode batch of 128 sequences x ctx ~1700 with Llama-3-8B's head layout: a 296-CTA balanced work plan over
    (sequence, kv head, page) with items cut across CTAs and merged inside the kernel.  Same geometry here on tiny other dims
    (tiny-llama-8bheads: 32 query heads / 8 kv heads / head_dim 128, llama3 RoPE scaling): 128 ragged prompts of 1600-1790 tokens through
    the scheduler (chunked prefill, 28 pages per sequence, positions past 1,700), 24 greedy tokens each; every 8th sequence — they are
    independent — is checked token for token against the oracle."""
    spec = O.PRESETS["tiny-llama-8bheads"]
    eng = Engine(spec.engine_json(num_pages=128 * 29 + 64, max_seq_len=1856, max_batch=128, max_step_tokens=8192, prefix_cache=0))
    rng = np.random.default_rng(2024)
    lens = rng.integers(1600, 1791, size=128)
    prompts = [rng.integers(0, spec.vocab, size=int(n)).astype(np.int32) for n in lens]
    G = 24
    tickets = [eng.tokens_submit(p.tolist(), G, flags=1) for p in prompts]
    outs = [eng.wait(t) for t in tickets]
    st = eng.stats()
    assert all(o.completion_tokens == G for o in outs) and st["decode_steps"] >= G - 1 and st["preemptions"] == 0
    assert st["pages_free"] == st["pages_total"]
    eng.close()
    orc = O.Oracle(spec, max_pos=1856, mode=1)
    checked = same = 0
    for i in list(range(0, 128, 8)) + [97, 127]:
        ref, margins, _ = orc.generate(prompts[i], G)
        k = 0
        while k < G and ref[k] == outs[i].token_ids[k]:
            k += 1
        assert k == G or margins[k] <= 2 * LOGIT_TOL, (i, int(lens[i]), k, float(margins[k]))
        checked += 1; same += k
    orc.close()
    print(f"batch geometry: {checked} sequences checked, {same}/{checked * G} tokens identical")


@pytest.mark.parametrize("name", CASES + ["tiny-llama-8bheads", "llama-3.2-1b"])
def test_cluster_splitk_projections_match_oracle_and_streamk(name):
    """sk_clusterk=7: qkv (+bias, RoPE, paged-KV write), o and down (+residual) as cluster split-K GEMMs with the reduction through distributed
    shared memory (gemm_clusterk.cu).  Cluster sizes 2, 3, 4 and 8 occur across these shapes (sk_clusterk_min_fill=0 lets the tiny ones
    through).  Against the oracle with the usual tolerance — and against the stream-K path: a different K split, so equal only up to fp32
    summation order (<= 1 bf16 ulp on O(1) logits)."""
    full = name == "llama-3.2-1b"
    spec = O.PRESETS[name]
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, min(spec.vocab, 256 if full else spec.vocab), size=n).astype(np.int32) for n in ((7, 100) if full else (1, 33, 128))]
    outs = {}
    for ck in (0, 7):
        kw = dict(sk_clusterk=ck, sk_clusterk_min_fill=0)
        if full:
            eng = Engine({"model": name, "num_pages": 64, "max_seq_len": 512, "max_batch": 8, "max_step_tokens": 512, "seed": spec.seed, **kw})
        else:
            _, eng = make_engine(name, **kw)
        logits = [eng.debug_prefill_logits(t) for t in prompts]
        gen = [list(eng.generate(p.tolist(), 12 if full else 24, flags=1).token_ids) for p in prompts] * 1
        gen2 = [list(eng.generate(p.tolist(), 12 if full else 24, flags=1).token_ids) for p in prompts]
        assert gen == gen2                                             # deterministic run to run (fixed reduction order)
        outs[ck] = (logits, gen)
        eng.close()
    for a, b in zip(outs[0][0], outs[7][0]):
        assert np.isfinite(b).all() and np.abs(a - b).max() < (0.2 if full else 2e-2)
    if not full:
        orc = O.Oracle(spec, max_pos=512, mode=1)
        for p, lg, g in zip(prompts, outs[7][0], outs[7][1]):
            assert np.abs(lg - orc.forward(p, all_logits=True)).max() < LOGIT_TOL
            ref, margins, _ = orc.generate(p, 24)
            k = 0
            while k < 24 and ref[k] == g[k]:
                k += 1
            assert k == 24 or margins[k] <= 2 * LOGIT_TOL, (k, margins[k])
        orc.close()


def test_router_keeps_conversations_on_the_replica_that_holds_their_prefix():
    """opsagent_b200/router.py over REAL engines (two replicas on this GPU): steps of one ReAct conversation — the history is resent every step,
    simple.go:498-501 — always reach the replica whose prefix cache holds the earlier steps' pages; new conversations spread; results equal a
    single engine's (greedy, same weights)."""
    from opsagent_b200.router import Router
    spec = O.PRESETS["tiny-llama"]
    cfg = spec.engine_json(num_pages=96, max_seq_len=1024, max_batch=8, max_step_tokens=256, prefix_cache=1)
    rt = Router.create(cfg, devices=[0, 0], max_inflight=8)
    solo = Engine(cfg)
    convs = {c: [("system", "You are a Kubernetes expert. " * 6), ("user", f"question number {c}: why is pod web-{c} crashing? " * 3)] for c in range(4)}
    home = {}
    for step in range(3):
        for c, msgs in convs.items():
            out = rt.chat_complete(spec.name, msgs, 8, flags=1)
            ref = solo.chat_complete(spec.name, msgs, 8, flags=1)
            assert list(out.token_ids) == list(ref.token_ids)
            r = rt.replica_of(msgs)
            assert home.setdefault(c, r) == r
            msgs += [("assistant", bytes(out.content).decode("latin-1")), ("user", "observation: NAME READY STATUS\nweb-0 0/1 CrashLoopBackOff " * 2)]
    st = rt.stats()
    assert sorted(st["routed"]) == [6, 6] and st["sticky_hits"] == 8                     # 4 conversations x 3 steps, 2 per replica, steps 2-3 sticky
    per = st["per_replica"]
    assert all(p["prefix_hit_tokens"] >= 2 * 2 * 64 for p in per)                          # later steps found their earlier pages on their home replica
    rt.close(); solo.close()



def test_native_front_routes_conversations_like_the_router_and_answers_like_one_engine():
    """csrc/http_server.cpp over two replicas on this GPU: concurrent HTTP conversations (ReAct: the history is resent every step) stay on their
    replica, new ones spread, a replica over its in-flight limit answers 429, and every completion equals a single engine's greedy result."""
    import json as _json
    import http.client
    import threading
    from opsagent_b200.native_front import NativeFront
    from opsagent_b200.router import Router
    spec = O.PRESETS["tiny-llama"]
    cfg = spec.engine_json(num_pages=96, max_seq_len=1024, max_batch=8, max_step_tokens=256, prefix_cache=1)
    rt = Router.create(cfg, devices=[0, 0])
    solo = Engine(cfg)
    front = NativeFront(rt.engines, max_inflight=8)

    def post(msgs, max_tokens=8):
        c = http.client.HTTPConnection("127.0.0.1", front.port, timeout=120)
        c.request("POST", "/v1/chat/completions", body=_json.dumps({"model": spec.name, "max_tokens": max_tokens, "messages": [{"role": r, "content": t} for r, t in msgs]}).encode(),
                  headers={"Authorization": "Bearer sk-local", "Content-Type": "application/json"})
        r = c.getresponse(); d = _json.loads(r.read()); c.close()
        return r.status, d
    convs = {c: [("system", "You are a Kubernetes expert. " * 6), ("user", f"question number {c}: why is pod web-{c} crashing? " * 3)] for c in range(4)}
    for step in range(3):
        res = {}

        def run(c):
            res[c] = post(convs[c])
        th = [threading.Thread(target=run, args=(c,)) for c in convs]
        [t.start() for t in th]; [t.join() for t in th]
        for c, msgs in convs.items():
            st, d = res[c]
            assert st == 200, d
            ref = solo.chat_complete(spec.name, msgs, 8, flags=0)
            want = bytes(ref.content).decode("utf-8", "replace").rstrip("\n")
            assert d["choices"][0]["message"]["content"] == want
            assert d["usage"]["prompt_tokens"] == ref.prompt_tokens and d["usage"]["completion_tokens"] == ref.completion_tokens
            msgs += [("assistant", want), ("user", "observation: NAME READY STATUS\nweb-0 0/1 CrashLoopBackOff " * 2)]
    st = front.stats()
    assert sum(st["routed"]) == 12 and st["sticky_hits"] == 8 and min(st["routed"]) >= 3      # 4 conversations x 3 steps; steps 2-3 sticky; both replicas used
    assert all(e["prefix_hit_tokens"] >= 64 for e in st["engines"])                          # later steps found their earlier pages on their home replica
    # admission control: 40 simultaneous long requests of ONE conversation all go to its home replica; more than max_inflight=8 at once -> some 429
    codes = []

    def flood():
        codes.append(post(convs[0], max_tokens=200)[0])
    th = [threading.Thread(target=flood) for _ in range(40)]
    [t.start() for t in th]; [t.join() for t in th]
    assert set(codes) <= {200, 429} and codes.count(200) >= 8 and codes.count(429) >= 1
    assert front.stats()["rejected_429"] == codes.count(429)
    front.shutdown(); rt.close(); solo.close()


def test_native_front_cancels_completions_of_clients_that_hang_up():
    """a caller that gives up (the reference's HTTP client timing out, a cancelled context) must not keep a decode slot and KV pages: the front notices
    the hang-up within one wait slice and calls oa_chat_cancel; the engine's own counter agrees and the pages come back"""
    import json as _json
    import socket
    import time
    from opsagent_b200.native_front import NativeFront
    spec, eng = make_engine("tiny-llama", max_seq_len=8192, num_pages=800, max_batch=8)
    front = NativeFront([eng])
    socks = []
    for k in range(6):          # six long completions (greedy on random weights mostly loops without ever emitting EOS; one that does simply finishes)
        body = _json.dumps({"model": spec.name, "max_tokens": 7000, "messages": [{"role": "user", "content": f"prompt number {k}: " + "describe the cluster " * (k + 1)}]}).encode()
        s = socket.create_connection(("127.0.0.1", front.port))
        s.sendall(b"POST /v1/chat/completions HTTP/1.1\r\nAuthorization: Bearer x\r\nContent-Length: " + str(len(body)).encode() + b"\r\n\r\n" + body)
        socks.append(s)
    time.sleep(0.2)
    for s in socks:
        s.close()
    t0 = time.time()
    while time.time() - t0 < 10 and front.stats()["connections"] > 0:
        time.sleep(0.05)
    st = front.stats()
    assert st["connections"] == 0 and st["cancelled"] >= 1, st
    assert st["engines"][0]["cancelled"] == st["cancelled"]
    assert time.time() - t0 < 3.0          # well before 7000 tokens would have been generated
    out = eng.chat_complete(spec.name, [("user", "still alive?")], 8, flags=1)      # the engine carries on, pages are back
    assert out.completion_tokens == 8
    es = eng.stats()
    assert es["running"] == 0 and es["waiting"] == 0 and es["pages_free"] >= es["pages_total"] - 16      # only prefix-cache pages of short prompts stay held
    front.shutdown(); eng.close()
