"""fp8 (e4m3) projection weights on the H100 (pytest -m gpu): the row quantiser and the W8A8 GEMMs through their C entry points against
torch, and the engine with "weight_dtype": "fp8_e4m3" against the oracle in mode 3 (tests/w8_fp8_ref.py: W8A8 projections with row-rule
scales), with the bounds of test_engine_gpu.py."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from opsagent_b200 import Engine, EngineError, _lib  # noqa: E402
from oracle import oracle as O  # noqa: E402  (checker only)
from w8_fp8_ref import W8Oracle  # noqa: E402  (checker only: the oracle in mode 3)

LOGIT_TOL = 2.5e-2
# Engine vs mode 3.  The mode-1 bound above does not carry over.  The engine and the oracle differ in summation order (and the fp8 tensor
# core sums a k block's 128 products with about 14 mantissa bits), so some bf16 activations differ by one ulp, as in mode 1; next to an e4m3
# rounding midpoint such a difference flips the element's e4m3 rounding, a full e4m3 step, and the next projection carries it on.  Measured on
# the tiny presets (H100): max 0.010-0.099, mean 0.002-0.017, against a quantisation effect (mode 3 vs mode 1) of max 0.07-0.22, mean
# 0.016-0.039.  So the bounds are 0.15 / 0.025, and the engine must be clearly closer to mode 3 than mode 3 is to mode 1.
W8_TOL_MAX, W8_TOL_MEAN = 0.15, 2.5e-2
FP8 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def L():
    return _lib.load()


def dev():
    return torch.device("cuda:0")


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def row_rule(x):
    """torch restatement of the row rule: (e4m3 bytes, fp32 scales) of the rows of x"""
    amax = x.float().abs().amax(dim=-1, keepdim=True).double()
    k = torch.ceil(torch.log2(torch.clamp(amax, min=1e-300) / 448.0))
    k = torch.where(amax > 448.0 * torch.exp2(k), k + 1, k)
    k = torch.where(amax <= 448.0 * torch.exp2(k - 1), k - 1, k)
    k = torch.where(amax == 0, torch.zeros_like(k), torch.clamp(k, min=-126))
    s = torch.exp2(k).float()
    return (x.float() / s).to(FP8).view(torch.uint8), s[..., 0]


def quant(L, x):
    R, Cc = x.shape
    q = torch.empty(R, Cc, dtype=torch.uint8, device=dev()); s = torch.empty(R, dtype=torch.float32, device=dev())
    assert L.oa_k_quant_rows_e4m3(ptr(x), ptr(q), ptr(s), R, Cc, None) == 0, _lib.last_error()
    return q, s


def deq(q, s):
    return q.view(FP8).float() * s[:, None]


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("R,Cc", [(1, 16), (37, 320), (128, 4096), (5, 14336), (300, 1024)])
def test_quantiser_matches_torch(L, R, Cc):
    g = torch.Generator(device="cpu").manual_seed(R + Cc)
    mag = 10.0 ** (torch.rand(R, 1, generator=g) * 16 - 8)                 # row maxima from 1e-8 to 1e8
    x = (torch.randn(R, Cc, generator=g) * mag).to(torch.bfloat16)
    x[0, :] = 0                                                            # all-zero row: s = 1, bytes 0
    if R > 3:
        x[1, :] = 0; x[1, 3] = 448.0                                       # amax = 448 * 2^0 exactly
        x[2, :] = 0; x[2, 5] = -448.0 * 2 ** -3; x[2, 6] = 1e-30           # tie at 2^-3, subnormal neighbours
        x[3, :] = 3.0e38                                                   # huge
    x = x.to(dev())
    q, s = quant(L, x)
    rq, rs = row_rule(x)
    assert torch.equal(s, rs)
    assert torch.equal(q, rq)
    assert not ((q == 0x7F) | (q == 0xFF)).any()


def _operands(M, N, K, seed, arbitrary_sw=False):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * (10.0 ** (torch.rand(M, 1, generator=g) * 4 - 2))).to(torch.bfloat16).to(dev())
    w = (torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16).to(dev())
    return a, w, g


def _weights8(L, w, arbitrary, g):
    if not arbitrary:
        return quant(L, w)
    # FP8-checkpoint style: any positive finite per-row scale (not a power of two), bytes e4m3(w / s)
    s = (w.float().abs().amax(dim=1) / 448.0 * (1.0 + torch.rand(w.shape[0], generator=g).to(dev()) * 0.7)).clamp(min=1e-12)
    return (w.float() / s[:, None]).to(FP8).view(torch.uint8).contiguous(), s.contiguous()


EPIS = {"store": 0, "resid": 1, "swiglu": 2}


# (N, K, block_n, persistent): K tails (320 = 2.5 k blocks), N tails (200 on 64-wide tiles); the persistent kernel runs 128-wide tiles
TILE_SHAPES = [(n, k, bn, p) for n, k, bn in [(256, 320, 128), (200, 256, 64), (1536, 1024, 128), (96, 4096, 32)] for p in (False, True)
               if bn == 128 or not p]


@pytest.mark.parametrize("arbitrary", [False, True])
@pytest.mark.parametrize("M", [1, 7, 128, 200, 1000])
@pytest.mark.parametrize("N,K,bn,persistent", TILE_SHAPES)
@pytest.mark.parametrize("epi", ["store", "resid", "swiglu"])
def test_gemm_fp8_tile_and_persistent(L, monkeypatch, epi, N, K, bn, persistent, M, arbitrary):
    if epi == "swiglu" and N % 32:
        return                                    # SwiGLU needs N % 32 == 0 (the interleave of 16 gate / 16 up rows)
    if persistent:
        monkeypatch.setenv("OA_GEMM_PERSISTENT_MIN_TILES", "1")
    else:
        monkeypatch.setenv("OA_GEMM_PERSISTENT_MIN_TILES", "1000000000")
    a, w, g = _operands(M, N, K, M * 7 + N + K)
    qa, sa = quant(L, a)
    qw, sw = _weights8(L, w, arbitrary, g)
    ref = deq(qa, sa).double() @ deq(qw, sw).double().T
    bias = (torch.randn(N, generator=g) * 0.1).to(torch.bfloat16).to(dev())
    resid = (torch.randn(M, N, generator=g)).to(torch.bfloat16).to(dev())
    out = torch.full((M, N // 2 if epi == "swiglu" else N), float("nan"), dtype=torch.bfloat16, device=dev())
    rc = L.oa_k_gemm_fp8(ptr(qa), ptr(sa), ptr(qw), ptr(sw), M, N, K, EPIS[epi], bn, ptr(out),
                         ptr(bias) if epi == "store" else None, ptr(resid) if epi == "resid" else None, None)
    assert rc == 0, _lib.last_error()
    if epi == "store":
        ref = ref + bias.double()
    elif epi == "resid":
        ref = ref + resid.double()
    else:
        r = ref.view(M, N // 32, 2, 16)
        gte, up = r[:, :, 0], r[:, :, 1]
        ref = (gte / (1 + torch.exp(-gte)) * up).reshape(M, N // 2)
    scale = ref.abs().max().item()
    err = (out.double() - ref).abs().max().item()
    assert torch.isfinite(out.float()).all()
    assert err <= 1e-2 * scale, (err, scale)


@pytest.mark.parametrize("arbitrary", [False, True])
@pytest.mark.parametrize("M", [1, 7, 128])
@pytest.mark.parametrize("N,K,bn,ctas", [(256, 320, 128, 132), (200, 256, 64, 37), (1536, 1024, 128, 132), (4096, 4096, 128, 132),
                                         (3072, 4096, 64, 100)])
def test_gemm_fp8_streamk(L, N, K, bn, ctas, M, arbitrary):
    a, w, g = _operands(M, N, K, M + N * 3 + K)
    qa, sa = quant(L, a)
    qw, sw = _weights8(L, w, arbitrary, g)
    ref = deq(qa, sa).double() @ deq(qw, sw).double().T
    out = torch.full((M, N), float("nan"), dtype=torch.float32, device=dev())
    assert L.oa_k_gemm_streamk_fp8(ptr(qa), ptr(sa), ptr(qw), ptr(sw), M, N, K, bn, ctas, 0, None, ptr(out), None) == 0, _lib.last_error()
    # the tensor core sums the 128 products of a k block with about 14 mantissa bits (measured up to 1.5e-4 of the output scale at K = 320,
    # M = 1); the promoted fp32 sum over blocks adds no more than fp32 rounding
    err = (out.double() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 5e-4, err
    # FUSE 2: x += product inside the GEMM, the stand-alone sum's bf16 result
    if bn == 128 and N % 32 == 0:
        x0 = torch.randn(M, N, generator=g).to(torch.bfloat16).to(dev())
        x = x0.clone()
        assert L.oa_k_gemm_streamk_fp8(ptr(qa), ptr(sa), ptr(qw), ptr(sw), M, N, K, bn, min(ctas, 132), 2, ptr(x), None, None) == 0, _lib.last_error()
        exp = (x0.float() + out).to(torch.bfloat16)
        assert torch.equal(x, exp)


def test_gemm_fp8_long_k_promotion(L):
    """Llama-3-8B's down projection (K = 14336) at M = 128: fp32 promotion per 128-wide k block keeps the sum to fp32 accuracy"""
    M, N, K = 128, 4096, 14336
    g = torch.Generator(device="cpu").manual_seed(1)
    a = (torch.rand(M, K, generator=g) * 2).to(torch.bfloat16).to(dev())          # SwiGLU-like inputs: mostly positive
    w = (torch.randn(N, K, generator=g) * 0.02 + 0.004).to(torch.bfloat16).to(dev())
    qa, sa = quant(L, a); qw, sw = quant(L, w)
    ref = deq(qa, sa).double() @ deq(qw, sw).double().T
    out = torch.empty(M, N, dtype=torch.float32, device=dev())
    assert L.oa_k_gemm_streamk_fp8(ptr(qa), ptr(sa), ptr(qw), ptr(sw), M, N, K, 128, 132, 0, None, ptr(out), None) == 0
    err_sk = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    o16 = torch.empty(M, N, dtype=torch.bfloat16, device=dev())
    assert L.oa_k_gemm_fp8(ptr(qa), ptr(sa), ptr(qw), ptr(sw), M, N, K, 0, 128, ptr(o16), None, None, None) == 0
    err_tile = ((o16.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"K=14336 max relative error: stream-K {err_sk:.3e}, tile kernel (bf16 output) {err_tile:.3e}")
    assert err_sk <= 1e-4, err_sk
    assert err_tile <= 2 ** -8 + 1e-4, err_tile          # bf16 output rounding on top


def test_gemm_fp8_refusals(L):
    a = torch.zeros(8, 64, dtype=torch.uint8, device=dev()); s = torch.ones(8, device=dev())
    out = torch.empty(8, 8, dtype=torch.bfloat16, device=dev())
    assert L.oa_k_gemm_fp8(ptr(a), ptr(s), ptr(a), ptr(s), 8, 8, 64, 3, 32, ptr(out), None, None, None) != 0      # no fp8 LM head
    assert L.oa_k_gemm_fp8(ptr(a), ptr(s), ptr(a), ptr(s), 8, 8, 64, 0, 256, ptr(out), None, None, None) != 0    # BN <= 128


# ------------------------------------------------------------------------------------------------ engine
def make_engine(name, **kw):
    spec = O.PRESETS[name]
    cfg = spec.engine_json(num_pages=64, max_seq_len=512, max_batch=16, max_step_tokens=256, weight_dtype="fp8_e4m3")
    cfg.update(kw)
    return spec, Engine(cfg)


CASES = ["tiny-llama", "tiny-llama-d128", "tiny-qwen", "tiny-llama-g8", "tiny-llama-mha"]


def _check_generation(ids, ref, margins):
    for i, (a, b) in enumerate(zip(ids, ref)):
        if a != b:
            assert margins[i] <= 2 * W8_TOL_MAX, f"token {i}: engine {a} reference {b} margin {margins[i]}"
            return
    assert list(ids) == list(ref)


def _check_logits(got, ref, what="", ref_mode1=None):
    assert np.isfinite(got).all()
    d = np.abs(got - ref)
    q = float(np.abs(ref - ref_mode1).mean()) if ref_mode1 is not None else float("nan")
    print(f"w8 logits {what}: max {d.max():.3e} mean {d.mean():.3e} (mode 3 vs mode 1: mean {q:.3e})")
    assert d.max() < W8_TOL_MAX and d.mean() < W8_TOL_MEAN, (what, float(d.max()), float(d.mean()))
    if ref_mode1 is not None:
        assert d.mean() < 0.7 * q, (what, float(d.mean()), q)


@pytest.mark.parametrize("name", CASES)
def test_engine_w8_matches_reference(name):
    spec, eng = make_engine(name)
    orc = W8Oracle(spec, max_pos=512)
    orc1 = O.Oracle(spec, max_pos=512, mode=1)
    rng = np.random.default_rng(1)
    for n in (1, 17, 64, 65, 150, 256):
        toks = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        _check_logits(eng.debug_prefill_logits(toks), orc.forward(toks, all_logits=True), f"{name} n={n}", orc1.forward(toks, all_logits=True))
    orc1.close()
    for n, g in ((5, 40), (70, 24), (130, 60)):
        prompt = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        ref, margins, _ = orc.generate(prompt, g)
        out = eng.generate(prompt.tolist(), g, flags=1)
        assert out.completion_tokens == g
        _check_generation(out.token_ids, ref, margins)
    st = eng.stats()
    assert st["weight_dtype"] == "fp8_e4m3" and st["kv_cache_dtype"] == "bf16" and eng.info["weight_dtype"] == "fp8_e4m3"
    eng.close(); orc.close()


def test_engine_w8_long_context_chunked_prefill_and_decode():
    spec, eng = make_engine("tiny-llama-d128", max_seq_len=8192, num_pages=200, max_step_tokens=2048, max_batch=4)
    orc = W8Oracle(spec, max_pos=5200)
    rng = np.random.default_rng(31)
    prompt = rng.integers(0, spec.vocab, size=5000).astype(np.int32)
    ref, margins, _ = orc.generate(prompt, 12)
    out = eng.generate(prompt.tolist(), 12, flags=1)
    _check_generation(out.token_ids, ref, margins)
    st = eng.stats()
    assert st["prefill_steps"] >= 3 and st["prefill_tokens"] == 5000
    eng.close(); orc.close()


@pytest.mark.parametrize("kv", ["bf16", "fp8_e4m3"])
def test_engine_w8_benchmarked_geometry_matches_reference(kv):
    """bench.py's geometry (tiny-llama-8bheads, 128 ragged sequences of 1600-1790 tokens, 24 greedy tokens each) with fp8 weights, alone and
    with the fp8 KV cache (modes 2 + 3)"""
    spec = O.PRESETS["tiny-llama-8bheads"]
    eng = Engine(spec.engine_json(num_pages=128 * 29 + 64, max_seq_len=1856, max_batch=128, max_step_tokens=8192, prefix_cache=0,
                                  weight_dtype="fp8_e4m3", kv_cache_dtype=kv))
    rng = np.random.default_rng(2024)
    lens = rng.integers(1600, 1791, size=128)
    prompts = [rng.integers(0, spec.vocab, size=int(n)).astype(np.int32) for n in lens]
    G = 24
    tickets = [eng.tokens_submit(p.tolist(), G, flags=1) for p in prompts]
    outs = [eng.wait(t) for t in tickets]
    st = eng.stats()
    assert all(o.completion_tokens == G for o in outs) and st["preemptions"] == 0 and st["pages_free"] == st["pages_total"]
    eng.close()
    orc = W8Oracle(spec, max_pos=1856, kv_fp8=kv == "fp8_e4m3")
    for i in list(range(0, 128, 16)) + [97, 127]:
        ref, margins, _ = orc.generate(prompts[i], G)
        _check_generation(outs[i].token_ids, ref, margins)
    orc.close()


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-llama-d128", "tiny-qwen"])
def test_engine_w8_fused_paths_agree_and_other_routes(name):
    """sk_fuse_epi 0 / 1 / 7 give bit-identical results (the scales are applied where each piece enters the fp32 tile); streamk = 0 (tile
    kernels only) and sk_max_rows = 256 (batches of 129-256 rows on the tile kernel with fp8) match the reference"""
    rng = np.random.default_rng(77)
    spec = O.PRESETS[name]
    prompts = [rng.integers(0, spec.vocab, size=n).astype(np.int32) for n in (1, 33, 128)]
    gen_prompts = [rng.integers(0, 256, size=n).astype(np.int32).tolist() for n in (3, 40, 90)]
    results = []
    for kw in (dict(sk_fuse_epi=0), dict(sk_fuse_epi=1), dict(sk_fuse_epi=7)):
        _, eng = make_engine(name, **kw)
        results.append(([eng.debug_prefill_logits(t) for t in prompts], [list(eng.generate(p, 20, flags=1).token_ids) for p in gen_prompts]))
        eng.close()
    for res in results[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(results[0][0], res[0]))
        assert results[0][1] == res[1]
    orc = W8Oracle(spec, max_pos=512)
    for kw in (dict(streamk=0), dict(sk_max_rows=256, max_batch=200, num_pages=220)):
        _, eng = make_engine(name, **kw)
        for p in gen_prompts:
            ref, margins, _ = orc.generate(np.array(p, np.int32), 20)
            _check_generation(eng.generate(p, 20, flags=1).token_ids, ref, margins)
        if "sk_max_rows" in kw:      # 160 concurrent sequences: decode steps of 129-256 rows
            ps = [rng.integers(0, spec.vocab, size=int(n)).astype(np.int32) for n in rng.integers(5, 40, size=160)]
            tickets = [eng.tokens_submit(p.tolist(), 8, 1) for p in ps]
            outs = [eng.wait(t) for t in tickets]
            for i in (0, 77, 159):
                ref, margins, _ = orc.generate(ps[i], 8)
                _check_generation(outs[i].token_ids, ref, margins)
        eng.close()
    orc.close()


def test_engine_w8_prefix_cache_concurrency_and_preemption():
    rng = np.random.default_rng(9)
    spec = O.PRESETS["tiny-llama"]
    orc = W8Oracle(spec, max_pos=256)
    base = rng.integers(0, 256, size=150).tolist()
    prompts = [base + rng.integers(0, 256, size=k).tolist() for k in (5, 20, 41, 3)]
    runs = []
    for pc in (0, 1):
        _, eng = make_engine("tiny-llama", prefix_cache=pc)
        runs.append([list(eng.generate(p, 16, flags=1).token_ids) for p in prompts])
        eng.close()
    assert runs[0] == runs[1]
    # concurrent requests (mixed prefill + decode steps)
    _, eng = make_engine("tiny-llama", max_step_tokens=128)
    tickets = [eng.tokens_submit(p, 16, 1) for p in prompts]
    for p, t in zip(prompts, tickets):
        ref, margins, _ = orc.generate(np.array(p, np.int32), 16)
        _check_generation(eng.wait(t).token_ids, ref, margins)
    assert eng.stats()["mixed_steps"] > 0
    eng.close()
    _, eng = make_engine("tiny-llama", num_pages=8, max_seq_len=256, max_batch=8)
    reqs = [rng.integers(0, spec.vocab, size=60).astype(np.int32) for _ in range(6)]
    tickets = [eng.tokens_submit(p.tolist(), 100, 1) for p in reqs]
    outs = [eng.wait(t) for t in tickets]
    for p, o in zip(reqs, outs):
        ref, margins, _ = orc.generate(p, 100)
        _check_generation(o.token_ids, ref, margins)
    st = eng.stats()
    assert st["preemptions"] > 0 and st["pages_free"] == st["pages_total"]
    eng.close(); orc.close()


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-qwen"])
def test_engine_w8_with_fp8_kv_cache(name):
    spec, eng = make_engine(name, kv_cache_dtype="fp8_e4m3")
    orc = W8Oracle(spec, max_pos=512, kv_fp8=True)
    rng = np.random.default_rng(4)
    for n in (17, 150):
        toks = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        _check_logits(eng.debug_prefill_logits(toks), orc.forward(toks, all_logits=True), f"{name} + fp8 KV n={n}")
    prompt = rng.integers(0, spec.vocab, size=40).astype(np.int32)
    ref, margins, _ = orc.generate(prompt, 30)
    _check_generation(eng.generate(prompt.tolist(), 30, flags=1).token_ids, ref, margins)
    st = eng.stats()
    assert st["weight_dtype"] == st["kv_cache_dtype"] == "fp8_e4m3"
    eng.close(); orc.close()


def test_engine_w8_memory():
    """weight_bytes is the real allocation (formula) and the default-sized pool gains what the smaller weights free"""
    for name in ("tiny-llama-d128", "llama-3-8b"):
        spec = O.PRESETS[name]
        qd, kd, H, F, V = spec.n_heads * spec.head_dim, spec.n_kv_heads * spec.head_dim, spec.hidden, spec.ffn, spec.vocab
        proj = (qd + 2 * kd) * H + H * qd + 3 * F * H
        rows = (qd + 2 * kd) + H + 2 * F + H
        head = 0 if spec.tie_embeddings else V * H * 2
        st = {}
        for dt in ("bf16", "fp8_e4m3"):
            extra = dict(kv_gb=2.0) if name == "llama-3-8b" else dict(kv_gb=0.25)
            cfg = spec.engine_json(max_seq_len=512, max_batch=16, max_step_tokens=256, weight_dtype=dt, **extra)
            eng = Engine(cfg)
            st[dt] = eng.stats()
            eng.close()
        want = {"bf16": (proj * 2) * spec.n_layers + V * H * 2 + head,
                "fp8_e4m3": (proj + 4 * rows) * spec.n_layers + V * H * 2 + head}
        for dt in st:
            assert st[dt]["weight_bytes"] == want[dt], (name, dt, st[dt]["weight_bytes"], want[dt])
            assert st[dt]["weight_dtype"] == dt
        assert st["bf16"]["pages_total"] == st["fp8_e4m3"]["pages_total"]          # a fixed kv_gb: same pool
    # default pool (what is free after the weights): the fp8 engine's pool is larger by about the freed bytes
    spec = O.PRESETS["llama-3-8b"]
    pools = {}
    for dt in ("bf16", "fp8_e4m3"):
        eng = Engine(spec.engine_json(max_seq_len=512, max_batch=16, max_step_tokens=256, weight_dtype=dt))
        pools[dt] = eng.stats()
        eng.close()
    freed = pools["bf16"]["weight_bytes"] - pools["fp8_e4m3"]["weight_bytes"]
    gained = pools["fp8_e4m3"]["kv_pool_bytes"] - pools["bf16"]["kv_pool_bytes"]
    print("llama-3-8b weight_bytes bf16 / fp8:", pools["bf16"]["weight_bytes"], pools["fp8_e4m3"]["weight_bytes"], "pool gained", gained)
    assert abs(gained - freed) < 0.05 * freed, (gained, freed)


# ------------------------------------------------------------------------------------------------ checkpoints
def _write(path, items):
    """items: list of (name, dtype, shape, raw bytes) -> *.safetensors"""
    header, blobs, off = {"__metadata__": {"format": "pt"}}, [], 0
    for name, dt, shape, raw in items:
        header[name] = {"dtype": dt, "shape": list(shape), "data_offsets": [off, off + len(raw)]}
        blobs.append(raw); off += len(raw)
    hj = json.dumps(header, separators=(",", ":")).encode(); hj += b" " * ((8 - len(hj) % 8) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(hj))); f.write(hj)
        for b in blobs:
            f.write(b)


PROJ = {"wq": "self_attn.q_proj", "wk": "self_attn.k_proj", "wv": "self_attn.v_proj", "wo": "self_attn.o_proj", "wg": "mlp.gate_proj",
        "wu": "mlp.up_proj", "wd": "mlp.down_proj"}


def _shapes(spec):
    H, qd, kd, F = spec.hidden, spec.n_heads * spec.head_dim, spec.n_kv_heads * spec.head_dim, spec.ffn
    return {"wq": (qd, H), "wk": (kd, H), "wv": (kd, H), "wo": (H, qd), "wg": (F, H), "wu": (F, H), "wd": (H, F)}


def _fp8_checkpoint(orc, path, q8, drop=(), override=None):
    """the oracle's checkpoint with every projection replaced by F8_E4M3 bytes + `_scale` tensors: q8[(layer, kind)] = (bytes [N, K] uint8,
    scale array, scale dtype, scale shape).  override: {name: (dtype, shape, raw)} replaces / adds entries"""
    tmp = path + ".bf16"
    O.write_safetensors(orc, tmp)
    raw = open(tmp, "rb").read(); os.remove(tmp)
    n = struct.unpack("<Q", raw[:8])[0]
    hdr = json.loads(raw[8:8 + n]); body = raw[8 + n:]
    items = []
    for name, meta in hdr.items():
        if name == "__metadata__":
            continue
        b, e = meta["data_offsets"]
        items.append([name, meta["dtype"], meta["shape"], body[b:e]])
    by = {it[0]: it for it in items}
    for (l, kind), (qb, sc, sdt, sshape) in q8.items():
        nm = f"model.layers.{l}.{PROJ[kind]}.weight"
        by[nm][1], by[nm][3] = "F8_E4M3", np.ascontiguousarray(qb).tobytes()
        if nm + "_scale" in drop:
            continue
        sraw = O.f32_to_bf16_bits(np.asarray(sc, np.float32)).tobytes() if sdt == "BF16" else np.asarray(sc, np.float32 if sdt == "F32" else np.float16).tobytes()
        items.append([nm + "_scale", sdt, sshape, sraw])
        items.append([f"model.layers.{l}.{PROJ[kind]}.input_scale", "F32", [], np.float32(0.5).tobytes()])     # ignored (dynamic scales)
    for nm, (dt, shape, r) in (override or {}).items():
        if nm in by:
            by[nm][1], by[nm][2], by[nm][3] = dt, shape, r
        else:
            items.append([nm, dt, shape, r])
    _write(path, items)


def test_checkpoints_fp8(L, tmp_path):
    name = "tiny-llama"
    spec = O.PRESETS[name]
    shapes = _shapes(spec)
    orc = O.Oracle(spec, max_pos=512, mode=1)
    rng = np.random.default_rng(3)
    toks = [rng.integers(0, spec.vocab, size=n).astype(np.int32) for n in (17, 150)]
    prompt = rng.integers(0, spec.vocab, size=40).astype(np.int32)
    _, seeded = make_engine(name)
    base = [seeded.debug_prefill_logits(t) for t in toks]
    base_gen = list(seeded.generate(prompt.tolist(), 24, flags=1).token_ids)
    seeded.close()
    # 1. the bytes and scales the engine derives from the seeded bf16 weights, as an F8_E4M3 checkpoint: bit-identical logits
    q8 = {}
    for l in range(spec.n_layers):
        for kind, shp in shapes.items():
            w = torch.from_numpy(orc.tensor(l, kind, shp).view(np.int16)).view(torch.bfloat16).to(dev())
            qb, sc = quant(L, w)
            q8[(l, kind)] = (qb.cpu().numpy(), sc.cpu().numpy()[:, None], "F32", [shp[0], 1])
    p1 = str(tmp_path / "derived.safetensors")
    _fp8_checkpoint(orc, p1, q8)
    _, eng = make_engine(name, weights=p1)
    for t, b in zip(toks, base):
        assert np.array_equal(eng.debug_prefill_logits(t), b)
    assert list(eng.generate(prompt.tolist(), 24, flags=1).token_ids) == base_gen
    eng.close()
    # 2. a bf16 checkpoint under weight_dtype fp8_e4m3 is quantised at load: the seeded run
    p2 = str(tmp_path / "bf16.safetensors")
    O.write_safetensors(orc, p2)
    _, eng = make_engine(name, weights=p2)
    for t, b in zip(toks, base):
        assert np.array_equal(eng.debug_prefill_logits(t), b)
    eng.close()
    # 3. arbitrary per-channel (F32 [N, 1], BF16 [N]) and per-tensor (F32 [], F16 [1]) scales against mode 3 on those weights
    m3 = W8Oracle(spec, max_pos=512)
    q8 = {}
    styles = [("F32", "row2"), ("BF16", "row1"), ("F32", "tensor0"), ("F16", "tensor1")]
    for l in range(spec.n_layers):
        for i, (kind, shp) in enumerate(shapes.items()):
            w = O._np_bf16_to_f32(orc.tensor(l, kind, shp))
            dt, style = styles[(i + l) % 4]
            amax = np.abs(w).max(axis=1) if style.startswith("row") else np.full(shp[0], np.abs(w).max())
            s = (amax / 448.0 * rng.uniform(1.0, 1.7, size=shp[0] if style.startswith("row") else 1)).astype(np.float32)
            s = np.broadcast_to(s, (shp[0],)).astype(np.float32)
            if dt == "BF16":
                s = O._np_bf16_to_f32(O.f32_to_bf16_bits(s))
            elif dt == "F16":
                s = s.astype(np.float16).astype(np.float32)
            qb = torch.from_numpy(w / s[:, None]).to(FP8).view(torch.uint8).numpy()
            sshape = {"row2": [shp[0], 1], "row1": [shp[0]], "tensor0": [], "tensor1": [1]}[style]
            q8[(l, kind)] = (qb, s if style.startswith("row") else s[:1], dt, sshape)
            m3.set_weight(l, kind, qb, s)
    p3 = str(tmp_path / "arbitrary.safetensors")
    _fp8_checkpoint(orc, p3, q8)
    _, eng = make_engine(name, weights=p3)
    for t in toks:
        _check_logits(eng.debug_prefill_logits(t), m3.forward(t, all_logits=True), "arbitrary-scale checkpoint")
    ref, margins, _ = m3.generate(prompt, 24)
    _check_generation(eng.generate(prompt.tolist(), 24, flags=1).token_ids, ref, margins)
    eng.close(); m3.close()
    # 4. malformed files are refused with a message naming the tensor
    l0q = "model.layers.0.self_attn.q_proj.weight"
    H, V = spec.hidden, spec.vocab
    bad = {
        "missing scale": (dict(drop=(l0q + "_scale",)), "q_proj.weight_scale"),
        "bad scale shape": (dict(override={l0q + "_scale": ("F32", [3], np.ones(3, np.float32).tobytes())}), "q_proj.weight_scale"),
        "negative scale": (dict(override={l0q + "_scale": ("F32", [], np.float32(-1).tobytes())}), "q_proj.weight_scale"),
        "nan scale": (dict(override={l0q + "_scale": ("F32", [1], np.float32(np.nan).tobytes())}), "q_proj.weight_scale"),
        "int scale": (dict(override={l0q + "_scale": ("I32", [], np.int32(1).tobytes())}), "q_proj.weight_scale"),
        "fp8 embedding": (dict(override={"model.embed_tokens.weight": ("F8_E4M3", [V, H], bytes(V * H))}), "embed_tokens"),
        "mixed q/k": (dict(override={"model.layers.1.self_attn.k_proj.weight": ("BF16", list(shapes["wk"]), bytes(2 * shapes["wk"][0] * H))}),
                      "must all be F8_E4M3 or none"),
    }
    for why, (kw, msg) in bad.items():
        p = str(tmp_path / f"bad_{why.replace(' ', '_').replace('/', '_')}.safetensors")
        _fp8_checkpoint(orc, p, q8, **kw)
        with pytest.raises(EngineError) as e:
            make_engine(name, weights=p)
        assert msg in str(e.value), (why, str(e.value))
    with pytest.raises(EngineError) as e:
        make_engine(name, weights=p3, weight_dtype="bf16")
    assert "_proj.weight" in str(e.value) and "weight_dtype fp8_e4m3" in str(e.value), str(e.value)
    orc.close()


K8S_BPE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bpe_k8s_8k.json")


def test_full_size_llama_3_2_1b_execute_prompt_w8_matches_oracle():
    """Llama-3.2-1B (seeded), POST /api/execute's messages through the Llama-3-format BPE, with fp8 weights.  The rule of the fp8-KV test:
    floor = the distance between the fp32 oracle (mode 0) and mode 3; the engine's logits at every prompt position must be within 1.5x that
    floor of the fp32 oracle (max and mean), and its 32 greedy tokens must equal mode 3's up to the first near-tie (margin <= 2x floor)."""
    from opsagent_b200 import workloads as WL
    name, n_new = "llama-3.2-1b", 32
    spec = O.PRESETS[name]
    msgs = [(m.Role, m.Content) for m in WL.execute_messages("execute how many namespace in the cluster?")]
    eng = Engine({"model": name, "num_pages": 64, "max_seq_len": 2048, "max_batch": 8, "max_step_tokens": 2048, "seed": spec.seed,
                  "tokenizer": K8S_BPE, "weight_dtype": "fp8_e4m3"})
    ids = eng.apply_chat_template(msgs)
    toks = np.array(ids, np.int32)
    got = eng.debug_prefill_logits(ids)
    out = eng.chat_complete(name, msgs, n_new, flags=1)
    eng.close()
    assert np.isfinite(got).all()
    orc0 = O.Oracle(spec, max_pos=len(ids) + n_new + 8, mode=0)
    ref0 = orc0.forward(toks, all_logits=True)
    orc0.close()
    orc3 = W8Oracle(spec, max_pos=len(ids) + n_new + 8)
    ref3_all = orc3.forward(toks, all_logits=True)
    floor_max, floor_mean = float(np.abs(ref3_all - ref0).max()), float(np.abs(ref3_all - ref0).mean())
    err_max, err_mean = float(np.abs(got - ref0).max()), float(np.abs(got - ref0).mean())
    lg = ref3_all[-1].copy()
    del ref3_all
    assert err_max <= 1.5 * floor_max + 1e-3 and err_mean <= 1.5 * floor_mean + 1e-4, (err_max, floor_max, err_mean, floor_mean)
    ref_t, margins = [], []
    for i in range(n_new):
        order = np.argsort(lg)
        ref_t.append(int(order[-1]) if lg[order[-1]] > lg[order[-2]] else int(min(order[-1], order[-2])))
        margins.append(float(abs(lg[order[-1]] - lg[order[-2]])))
        if i + 1 < n_new:
            lg = orc3.forward(np.array([ref_t[-1]], np.int32), pos0=len(ids) + i)[0]
    orc3.close()
    k = 0
    while k < n_new and out.token_ids[k] == ref_t[k]:
        k += 1
    assert k == n_new or margins[k] <= 2 * floor_max, (k, margins[k], floor_max)
    print("llama-3.2-1b w8:", {"prompt_tokens": len(ids), "err_max": err_max, "err_mean": err_mean, "floor_max": floor_max,
                               "floor_mean": floor_mean, "same_tokens": k})
