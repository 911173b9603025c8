"""fp8 (e4m3) paged KV cache on the H100 (pytest -m gpu): the fp8 attention kernels and the KV writer through their C entry points, and
the engine with "kv_cache_dtype": "fp8_e4m3" against the oracle in mode 2 (tests/kv_fp8_ref.py: mode 1 with the cache holding
e4m3(x / s) * s), with the bounds of test_engine_gpu.py."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from kv_fp8_ref import Fp8Oracle  # noqa: E402  (checker only: the oracle in mode 2)
from opsagent_b200 import Engine, EngineError, _lib  # noqa: E402
from oracle import oracle as O  # noqa: E402  (checker only)

LOGIT_TOL = 2.5e-2
FP8 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def L():
    return _lib.load()


def dev():
    return torch.device("cuda:0")


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def q8(x, s):
    """bytes the writers store for x (fp32 math): e4m3(x * (1/s)), saturating"""
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(s, dtype=torch.float32)
    return (x.float() * inv.to(x.device)).clamp(-448, 448).to(FP8)


def _attn_ref(q, kcache, vcache, bt, ctx, qlens, nh, nkv, D):
    """fp32 paged causal GQA attention (the reference of tests/test_kernels_gpu.py).  caches [pages, nkv, 64, D]"""
    grp = nh // nkv
    outs, row = [], 0
    for i, (c, ql) in enumerate(zip(ctx, qlens)):
        pages = bt[i, : (c + 63) // 64]
        K = kcache[pages].permute(0, 2, 1, 3).reshape(-1, nkv, D)[:c].float()
        V = vcache[pages].permute(0, 2, 1, 3).reshape(-1, nkv, D)[:c].float()
        qi = q[row:row + ql].float()
        Kh = K.repeat_interleave(grp, dim=1); Vh = V.repeat_interleave(grp, dim=1)
        s = torch.einsum("qhd,khd->hqk", qi, Kh) / (D ** 0.5)
        qpos = torch.arange(c - ql, c, device=q.device)[:, None]; kpos = torch.arange(c, device=q.device)[None, :]
        s = s.masked_fill((kpos > qpos)[None], float("-inf"))
        outs.append(torch.einsum("hqk,khd->qhd", torch.softmax(s, dim=-1), Vh)); row += ql
    return torch.cat(outs, 0)


def _fp8_cache(num_pages, nkv, D, seed, ks, vs, mag=1.0):
    """-> (byte cache [2, pages, nkv, 64*D] in the fp8 layout, dequantised K and V [pages, nkv, 64, D])"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    kv = (torch.randn(2, num_pages, nkv, 64, D, generator=g) * mag).to(torch.bfloat16).to(dev())
    k8, v8 = q8(kv[0], ks), q8(kv[1], vs)
    cache = torch.stack([k8.view(torch.uint8).reshape(num_pages, nkv, 64 * D),
                         v8.view(torch.uint8).transpose(2, 3).contiguous().reshape(num_pages, nkv, 64 * D)])
    return cache.contiguous(), k8.float() * ks, v8.float() * vs


def _tables(ctx, maxp, num_pages, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    perm = torch.randperm(num_pages, generator=g)
    bt = torch.zeros(len(ctx), maxp, dtype=torch.int32); k = 0
    for i, c in enumerate(ctx):
        npg = (c + 63) // 64; bt[i, :npg] = perm[k:k + npg].to(torch.int32); k += npg
    return bt, g


SCALES = [(1.0, 1.0), (0.37, 2.9)]


@pytest.mark.parametrize("ks,vs", SCALES)
@pytest.mark.parametrize("splits", [0, 3])
@pytest.mark.parametrize("nh,nkv,D", [(32, 8, 128), (8, 2, 64), (5, 1, 64), (8, 1, 128), (40, 8, 128), (4, 4, 64)])
def test_fp8_paged_decode_attention(L, nh, nkv, D, splits, ks, vs):
    ctx = [1, 63, 64, 65, 200, 1000, 129, 517]
    n = len(ctx); maxp = 20; num_pages = 150
    cache, kd, vd = _fp8_cache(num_pages, nkv, D, 11, ks, vs, mag=2.0 * ks)
    bt, g = _tables(ctx, maxp, num_pages, 5)
    q = torch.randn(n, nh, D, generator=g).to(torch.bfloat16).to(dev())
    out = torch.full((n, nh, D), float("nan"), dtype=torch.bfloat16, device=dev())
    ctx_a = np.array(ctx, np.int32); ql = np.ones(n, np.int32); bt_np = np.ascontiguousarray(bt.numpy())
    rc = L.oa_k_paged_attention_fp8(ptr(q), ptr(out), ptr(cache), num_pages, bt_np.ctypes.data, maxp, ctx_a.ctypes.data, ql.ctypes.data, n,
                                    nh, nkv, D, splits, ks, vs, None)
    assert rc == 0, _lib.last_error()
    ref = _attn_ref(q, kd, vd, bt.to(dev()).long(), ctx, [1] * n, nh, nkv, D) / vs
    assert torch.isfinite(out.float()).all()
    err = (out.float() / vs - ref).abs().max().item()      # compared in units of the V scale
    assert err < 2e-2, err


@pytest.mark.parametrize("ks,vs", SCALES)
@pytest.mark.parametrize("nh,nkv,D", [(8, 2, 128), (4, 2, 64), (5, 1, 64), (8, 1, 128), (4, 4, 64)])
def test_fp8_paged_prefill_attention(L, nh, nkv, D, ks, vs):
    cases = [(64, 64), (130, 130), (200, 37), (1, 1), (333, 100), (128, 128)]
    ctx = [c for c, _ in cases]; qlens = [q for _, q in cases]
    n = len(ctx); maxp = 8; num_pages = 40
    cache, kd, vd = _fp8_cache(num_pages, nkv, D, 3, ks, vs, mag=2.0 * ks)
    bt, g = _tables(ctx, maxp, num_pages, 9)
    T = sum(qlens)
    q = torch.randn(T, nh, D, generator=g).to(torch.bfloat16).to(dev())
    out = torch.full((T, nh, D), float("nan"), dtype=torch.bfloat16, device=dev())
    ctx_a = np.array(ctx, np.int32); ql = np.array(qlens, np.int32); bt_np = np.ascontiguousarray(bt.numpy())
    rc = L.oa_k_paged_attention_fp8(ptr(q), ptr(out), ptr(cache), num_pages, bt_np.ctypes.data, maxp, ctx_a.ctypes.data, ql.ctypes.data, n,
                                    nh, nkv, D, 0, ks, vs, None)
    assert rc == 0, _lib.last_error()
    ref = _attn_ref(q, kd, vd, bt.to(dev()).long(), ctx, qlens, nh, nkv, D) / vs
    assert torch.isfinite(out.float()).all()
    err = (out.float() / vs - ref).abs().max().item()
    assert err < 2e-2, err


def _rope_tables(D, max_pos, theta=500000.0):
    half = D // 2
    inv = theta ** (-2.0 * torch.arange(half, dtype=torch.float64) / D)
    a = torch.arange(max_pos, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.cos(a).float().to(dev()).contiguous(), torch.sin(a).float().to(dev()).contiguous()


@pytest.mark.parametrize("ks,vs", SCALES)
@pytest.mark.parametrize("nh,nkv,D", [(8, 2, 128), (5, 1, 64)])
def test_fp8_kv_write(L, nh, nkv, D, ks, vs):
    T, num_pages, max_pos = 150, 12, 512
    g = torch.Generator(device="cpu").manual_seed(D + nh)
    qkv = (torch.randn(T, (nh + 2 * nkv) * D, generator=g) * 3).to(torch.bfloat16).to(dev())
    pos = torch.randint(0, max_pos, (T,), generator=g, dtype=torch.int32).to(dev())
    slots = torch.randperm(num_pages * 64, generator=g)[:T].to(torch.int32).to(dev())
    cs, sn = _rope_tables(D, max_pos)
    q_out = torch.empty(T, nh * D, dtype=torch.bfloat16, device=dev())
    cache = torch.full((2, num_pages, nkv, 64 * D), 0x7F, dtype=torch.uint8, device=dev())    # NaN bytes: every written byte must change
    assert L.oa_k_kv_write_fp8(ptr(qkv), ptr(pos), ptr(slots), ptr(cs), ptr(sn), ptr(q_out), ptr(cache), num_pages, T, nh, nkv, D, ks, vs, None) == 0
    half = D // 2
    x = qkv.float().view(T, nh + 2 * nkv, D)
    c, s = cs[pos.long()][:, None, :], sn[pos.long()][:, None, :]
    lo, hi = x[..., :half], x[..., half:]
    rot = torch.cat([lo * c - hi * s, hi * c + lo * s], dim=-1).to(torch.bfloat16)        # fp32 RoPE -> bf16
    assert ((q_out.float().view(T, nh, D) - rot[:, :nh].float()).abs() <= rot[:, :nh].float().abs() * 2.0 ** -7 + 1e-6).all()
    page, off = (slots.long() // 64), (slots.long() % 64)
    kb = cache[0].view(num_pages, nkv, 64, D)[page, :, off]                           # [T, nkv, D]: K as [token][D]
    vb = cache[1].view(num_pages, nkv, D, 64)[page, :, :, off]                        # [T, nkv, D]: V transposed as [D][token]
    v_ref = q8(x[:, nh + nkv:].to(torch.bfloat16), vs).view(torch.uint8)
    assert torch.equal(vb, v_ref)                                                      # V: bit-exact
    # K: the kernel's fp32 RoPE may contract to FMA, so its bf16 value is torch's or a bf16 neighbour.  Where all three give the same byte the
    # kernel's byte must be exactly that one; everywhere it must be one of the three
    kr = rot[:, nh:nh + nkv]
    lo_n, hi_n = torch.nextafter(kr, torch.full_like(kr, -float("inf"))), torch.nextafter(kr, torch.full_like(kr, float("inf")))
    b0, b1, b2 = (q8(t, ks).view(torch.uint8) for t in (kr, lo_n, hi_n))
    unambiguous = (b0 == b1) & (b0 == b2)
    assert unambiguous.float().mean() > 0.8          # measured 0.87-0.88: a bf16 step crosses an e4m3 rounding boundary for the rest
    assert torch.equal(kb[unambiguous], b0[unambiguous])
    assert ((kb == b0) | (kb == b1) | (kb == b2)).all()
    # nothing outside the written rows changed
    written = torch.zeros(num_pages, 64, dtype=torch.bool, device=dev()); written[page, off] = True
    assert (cache[0].view(num_pages, nkv, 64, D).permute(0, 2, 1, 3)[~written] == 0x7F).all()
    assert (cache[1].view(num_pages, nkv, D, 64).permute(0, 3, 1, 2)[~written] == 0x7F).all()


# ------------------------------------------------------------------------------------------------ engine
def make_engine(name, **kw):
    spec = O.PRESETS[name]
    cfg = spec.engine_json(num_pages=64, max_seq_len=512, max_batch=16, max_step_tokens=256, kv_cache_dtype="fp8_e4m3")
    cfg.update(kw)
    return spec, Engine(cfg)


CASES = ["tiny-llama", "tiny-llama-d128", "tiny-qwen", "tiny-llama-g8", "tiny-llama-mha"]


def _check_generation(ids, ref, margins):
    for i, (a, b) in enumerate(zip(ids, ref)):
        if a != b:
            assert margins[i] <= 2 * LOGIT_TOL, f"token {i}: engine {a} reference {b} margin {margins[i]}"
            return
    assert list(ids) == list(ref)


@pytest.mark.parametrize("name", CASES)
def test_engine_fp8_matches_reference(name):
    spec, eng = make_engine(name)
    orc = Fp8Oracle(spec, max_pos=512)
    rng = np.random.default_rng(1)
    for n in (1, 17, 64, 65, 150, 256):
        toks = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        got = eng.debug_prefill_logits(toks)
        ref = orc.forward(toks, all_logits=True)
        assert np.isfinite(got).all()
        err = np.abs(got - ref).max()
        assert err < LOGIT_TOL, (n, err)
    for n, g in ((5, 40), (70, 24), (130, 60)):
        prompt = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        ref, margins, _ = orc.generate(prompt, g)
        out = eng.generate(prompt.tolist(), g, flags=1)
        assert out.completion_tokens == g
        _check_generation(out.token_ids, ref, margins)
    st = eng.stats()
    assert st["kv_cache_dtype"] == "fp8_e4m3"
    eng.close(); orc.close()


def test_engine_fp8_long_context_chunked_prefill_and_decode():
    spec, eng = make_engine("tiny-llama-d128", max_seq_len=8192, num_pages=200, max_step_tokens=2048, max_batch=4)
    orc = Fp8Oracle(spec, max_pos=5200)
    rng = np.random.default_rng(31)
    prompt = rng.integers(0, spec.vocab, size=5000).astype(np.int32)
    ref, margins, _ = orc.generate(prompt, 12)
    out = eng.generate(prompt.tolist(), 12, flags=1)
    _check_generation(out.token_ids, ref, margins)
    st = eng.stats()
    assert st["prefill_steps"] >= 3 and st["prefill_tokens"] == 5000
    eng.close(); orc.close()


def test_engine_fp8_benchmarked_geometry_matches_reference():
    """128 ragged sequences of 1600-1790 tokens on Llama-3-8B's attention geometry (tiny-llama-8bheads): the 296-CTA decode work plan with
    cut items and in-kernel merges that bench.py times, 24 greedy tokens each; every 8th sequence (they are independent) and two more are
    checked token for token against the mode-2 oracle, as test_benchmarked_batch_geometry_matches_oracle does for bf16"""
    spec = O.PRESETS["tiny-llama-8bheads"]
    eng = Engine(spec.engine_json(num_pages=128 * 29 + 64, max_seq_len=1856, max_batch=128, max_step_tokens=8192, prefix_cache=0,
                                  kv_cache_dtype="fp8_e4m3"))
    rng = np.random.default_rng(2024)
    lens = rng.integers(1600, 1791, size=128)
    prompts = [rng.integers(0, spec.vocab, size=int(n)).astype(np.int32) for n in lens]
    G = 24
    tickets = [eng.tokens_submit(p.tolist(), G, flags=1) for p in prompts]
    outs = [eng.wait(t) for t in tickets]
    st = eng.stats()
    assert all(o.completion_tokens == G for o in outs) and st["preemptions"] == 0 and st["pages_free"] == st["pages_total"]
    eng.close()
    orc = Fp8Oracle(spec, max_pos=1856)
    for i in list(range(0, 128, 8)) + [97, 127]:
        ref, margins, _ = orc.generate(prompts[i], G)
        _check_generation(outs[i].token_ids, ref, margins)
    orc.close()


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-llama-d128"])
def test_engine_fp8_fused_and_cluster_paths_agree(name):
    """every KV writer stores through one helper: the fused stream-K and cluster split-K qkv epilogues give the unfused results exactly"""
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
    _, eng = make_engine(name, sk_clusterk=7, sk_clusterk_min_fill=0)
    orc = Fp8Oracle(spec, max_pos=512)
    for p in gen_prompts:
        ref, margins, _ = orc.generate(np.array(p, np.int32), 20)
        _check_generation(eng.generate(p, 20, flags=1).token_ids, ref, margins)
    eng.close(); orc.close()


def test_engine_fp8_prefix_cache_concurrency_and_preemption():
    rng = np.random.default_rng(9)
    spec = O.PRESETS["tiny-llama"]
    orc = Fp8Oracle(spec, max_pos=256)
    base = rng.integers(0, 256, size=150).tolist()
    prompts = [base + rng.integers(0, 256, size=k).tolist() for k in (5, 20, 41, 3)]
    runs = []
    for pc in (0, 1):          # reused pages hold the same bytes as recomputed ones
        _, eng = make_engine("tiny-llama", prefix_cache=pc)
        runs.append([list(eng.generate(p, 16, flags=1).token_ids) for p in prompts])
        eng.close()
    assert runs[0] == runs[1]
    # concurrent requests (mixed prefill + decode steps): each gets what the reference gives it alone, up to near-ties
    _, eng = make_engine("tiny-llama", max_step_tokens=128)
    tickets = [eng.tokens_submit(p, 16, 1) for p in prompts]
    for p, t in zip(prompts, tickets):
        ref, margins, _ = orc.generate(np.array(p, np.int32), 16)
        _check_generation(eng.wait(t).token_ids, ref, margins)
    eng.close()
    # a pool too small for all requests at once: sequences are preempted (recompute) and still finish right
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


def test_engine_fp8_pool_holds_twice_the_pages():
    spec = O.PRESETS["tiny-llama-d128"]
    counts = {}
    for dt in ("bf16", "fp8_e4m3"):
        eng = Engine(spec.engine_json(kv_gb=0.25, max_seq_len=512, max_batch=16, max_step_tokens=256, kv_cache_dtype=dt))
        st = eng.stats()
        counts[dt] = st["pages_total"]
        assert st["kv_cache_dtype"] == dt
        assert eng.info["kv_bytes_per_token"] == 2 * spec.n_layers * spec.n_kv_heads * spec.head_dim * (1 if dt == "fp8_e4m3" else 2)
        eng.close()
    assert abs(counts["fp8_e4m3"] - 2 * counts["bf16"]) <= 1, counts


def _write_checkpoint(orc, path, scales=None, extra=None):
    """the oracle's tensors (test_engine_gpu's writer) plus optional KV scale tensors: scales = {name: (dtype, shape, values)}"""
    O.write_safetensors(orc, path)
    if not scales:
        return
    raw = open(path, "rb").read()
    n = struct.unpack("<Q", raw[:8])[0]
    hdr = json.loads(raw[8:8 + n]); body = bytearray(raw[8 + n:])
    for name, (dt, shape, vals) in scales.items():
        a = np.asarray(vals, {"F32": np.float32, "F16": np.float16}.get(dt, np.float32))
        b = (O.f32_to_bf16_bits(a.astype(np.float32)).tobytes() if dt == "BF16" else a.tobytes())
        hdr[name] = {"dtype": dt, "shape": shape, "data_offsets": [len(body), len(body) + len(b)]}
        body += b
    hj = json.dumps(hdr, separators=(",", ":")).encode(); hj += b" " * ((8 - len(hj) % 8) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(hj))); f.write(hj); f.write(bytes(body))


def test_checkpoint_kv_scales(tmp_path):
    name = "tiny-llama"
    spec = O.PRESETS[name]
    orc = O.Oracle(spec, max_pos=512, mode=1)
    ks, vs = [0.37, 1.5], [2.9, 0.75]
    sc = {}
    for l in range(spec.n_layers):
        sc[f"model.layers.{l}.self_attn.k_scale"] = ("F32", [], [ks[l]])
        sc[f"model.layers.{l}.self_attn.v_scale"] = ("BF16" if l else "F16", [1], [vs[l]])
    path = str(tmp_path / "m.safetensors")
    _write_checkpoint(orc, path, sc)
    # the engine reads the scale tensors back from the checkpoint: the reference gets the values as stored
    ks_s = [np.float32(ks[0]), np.float32(ks[1])]
    vs_s = [float(np.float16(vs[0])), float(O._np_bf16_to_f32(O.f32_to_bf16_bits(np.float32(vs[1])))[0])]
    _, eng = make_engine(name, weights=path)
    m2 = Fp8Oracle(spec, max_pos=512, k_scale=ks_s, v_scale=vs_s)
    rng = np.random.default_rng(3)
    for n in (17, 150):
        toks = rng.integers(0, spec.vocab, size=n).astype(np.int32)
        assert np.abs(eng.debug_prefill_logits(toks) - m2.forward(toks, all_logits=True)).max() < LOGIT_TOL
    prompt = rng.integers(0, spec.vocab, size=40).astype(np.int32)
    ref, margins, _ = m2.generate(prompt, 24)
    _check_generation(eng.generate(prompt.tolist(), 24, flags=1).token_ids, ref, margins)
    eng.close(); m2.close()
    # a bf16 cache ignores the scales
    _, eng = make_engine(name, weights=path, kv_cache_dtype="bf16")
    toks = rng.integers(0, spec.vocab, size=33).astype(np.int32)
    assert np.abs(eng.debug_prefill_logits(toks) - orc.forward(toks, all_logits=True)).max() < LOGIT_TOL
    eng.close()
    bad = {
        "negative": {**sc, "model.layers.0.self_attn.k_scale": ("F32", [], [-1.0])},
        "nan": {**sc, "model.layers.1.self_attn.v_scale": ("F32", [1], [float("nan")])},
        "some layers only": {k: v for k, v in sc.items() if not k.startswith("model.layers.1.")},
        "wrong shape": {**sc, "model.layers.0.self_attn.v_scale": ("F32", [2], [1.0, 1.0])},
    }
    for why, s in bad.items():
        p = str(tmp_path / f"bad_{why.replace(' ', '_')}.safetensors")
        _write_checkpoint(orc, p, s)
        with pytest.raises(EngineError) as e:
            make_engine(name, weights=p)
        assert "scale" in str(e.value), (why, str(e.value))
    orc.close()


K8S_BPE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bpe_k8s_8k.json")


def test_full_size_llama_3_2_1b_execute_prompt_fp8_matches_oracle():
    """Llama-3.2-1B (seeded), POST /api/execute's exact messages through the Llama-3-format BPE, with the fp8 cache.  At full size the bf16
    rounding of every stored activation, and here the e4m3 rounding of K and V, move two computations apart chaotically with depth, so the
    tolerance is relative to a measured floor (the rule of test_engine_gpu.py's _full_size_parity): floor = the distance between the fp32
    oracle (mode 0) and the oracle in mode 2; the engine's logits at every prompt position must be within 1.5x that floor of the fp32
    oracle (max and mean), and its 32 greedy tokens must equal mode 2's wherever the margin exceeds 2x the floor."""
    from opsagent_b200 import workloads as WL
    name, n_new = "llama-3.2-1b", 32
    spec = O.PRESETS[name]
    msgs = [(m.Role, m.Content) for m in WL.execute_messages("execute how many namespace in the cluster?")]
    eng = Engine({"model": name, "num_pages": 64, "max_seq_len": 2048, "max_batch": 8, "max_step_tokens": 2048, "seed": spec.seed,
                  "tokenizer": K8S_BPE, "kv_cache_dtype": "fp8_e4m3"})
    ids = eng.apply_chat_template(msgs)
    toks = np.array(ids, np.int32)
    got = eng.debug_prefill_logits(ids)
    out = eng.chat_complete(name, msgs, n_new, flags=1)
    eng.close()
    assert np.isfinite(got).all()
    orc0 = O.Oracle(spec, max_pos=len(ids) + n_new + 8, mode=0)
    ref0 = orc0.forward(toks, all_logits=True)
    orc0.close()
    orc2 = Fp8Oracle(spec, max_pos=len(ids) + n_new + 8)
    ref2_all = orc2.forward(toks, all_logits=True)
    floor_max, floor_mean = float(np.abs(ref2_all - ref0).max()), float(np.abs(ref2_all - ref0).mean())
    err_max, err_mean = float(np.abs(got - ref0).max()), float(np.abs(got - ref0).mean())
    lg = ref2_all[-1].copy()
    del ref2_all
    assert err_max <= 1.5 * floor_max + 1e-3 and err_mean <= 1.5 * floor_mean + 1e-4, (err_max, floor_max, err_mean, floor_mean)
    ref_t, margins = [], []
    for i in range(n_new):          # greedy continuation from the KV state the prefill left in the oracle
        order = np.argsort(lg)
        ref_t.append(int(order[-1]) if lg[order[-1]] > lg[order[-2]] else int(min(order[-1], order[-2])))
        margins.append(float(abs(lg[order[-1]] - lg[order[-2]])))
        if i + 1 < n_new:
            lg = orc2.forward(np.array([ref_t[-1]], np.int32), pos0=len(ids) + i)[0]
    orc2.close()
    k = 0
    while k < n_new and out.token_ids[k] == ref_t[k]:
        k += 1
    assert k == n_new or margins[k] <= 2 * floor_max, (k, margins[k], floor_max)
    print("llama-3.2-1b fp8:", {"prompt_tokens": len(ids), "err_max": err_max, "err_mean": err_mean, "floor_max": floor_max,
                                "floor_mean": floor_mean, "same_tokens": k})
