"""fp8 (e4m3) projection weights, CPU side: the weight_dtype option as the host parses it, the decode byte model, and the oracle's mode 3
(tests/w8_fp8_oracle.c: W8A8 projections with row-rule scales), which the GPU tests hold the engine to."""
import ctypes as C
import json

import numpy as np
import pytest

from kv_fp8_ref import Fp8Oracle
from opsagent_b200 import _lib
from oracle import oracle as O
from w8_fp8_ref import W8Oracle, lib as w8lib, w8_row

torch = pytest.importorskip("torch")


def _model_info(cfg):
    L = _lib.load()
    buf = C.create_string_buffer(2048)
    rc = L.oa_host_model_info(json.dumps(cfg).encode(), buf, 2048)
    return rc, (json.loads(buf.value.decode()) if rc == 0 else None)


def _w8_bytes(spec_or_name) -> float:
    """decode weight bytes with fp8 projections: 1 B per projection element + one fp32 scale per output row, the rest bf16"""
    s = O.PRESETS[spec_or_name]
    qd, kd = s.n_heads * s.head_dim, s.n_kv_heads * s.head_dim
    proj = (qd + 2 * kd) * s.hidden + s.hidden * qd + 3 * s.ffn * s.hidden
    rows = (qd + 2 * kd) + s.hidden + 2 * s.ffn + s.hidden
    other = 2 * s.hidden + ((qd + 2 * kd) if s.qkv_bias else 0)
    return float((proj + 4 * rows + 2 * other) * s.n_layers + 2 * (s.hidden + s.vocab * s.hidden))


@pytest.mark.parametrize("name", ["llama-3-8b", "llama-3.2-1b", "qwen2.5-32b", "tiny-llama", "tiny-qwen"])
def test_model_info_reports_fp8_weights(name):
    cfg = {"model": name} if name in O.PRESETS and not name.startswith("tiny") else O.PRESETS[name].engine_json()
    rc, base = _model_info(cfg)
    assert rc == 0 and "weight_dtype" not in base                 # default output as before
    rc, bf = _model_info({**cfg, "weight_dtype": "bf16"})
    assert rc == 0 and bf == base
    rc, f8 = _model_info({**cfg, "weight_dtype": "fp8_e4m3"})
    assert rc == 0 and f8["weight_dtype"] == "fp8_e4m3"
    assert f8["decode_weight_bytes"] == _w8_bytes(name)
    assert f8["kv_bytes_per_token"] == base["kv_bytes_per_token"]
    rc, both = _model_info({**cfg, "weight_dtype": "fp8_e4m3", "kv_cache_dtype": "fp8_e4m3"})
    assert rc == 0 and both["weight_dtype"] == both["kv_cache_dtype"] == "fp8_e4m3"
    assert both["decode_weight_bytes"] == f8["decode_weight_bytes"] and both["kv_bytes_per_token"] * 2 == base["kv_bytes_per_token"]
    if name == "llama-3-8b":
        assert abs(base["decode_weight_bytes"] / 1e9 - 15.010) < 0.02          # unchanged bf16 byte model
        assert abs(f8["decode_weight_bytes"] / 1e9 - 8.04) < 0.01               # 6.98 GB e4m3 + 1.05 GB LM head + 5.5 MB scales


@pytest.mark.parametrize("cfg, msg", [
    ({"weight_dtype": "fp8"}, "weight_dtype must be bf16 or fp8_e4m3"),
    ({"weight_dtype": "FP8_E4M3"}, "weight_dtype must be bf16 or fp8_e4m3"),
    ({"weight_dtype": "e4m3"}, "weight_dtype must be bf16 or fp8_e4m3"),
    ({"weight_dtype": ""}, "weight_dtype must be bf16 or fp8_e4m3"),
    ({"weight_dtype": "fp8_e4m3", "tp": 2}, "needs tp = 1"),
    ({"weight_dtype": "fp8_e4m3", "tp": 2, "tp_rank": 1}, "needs tp = 1"),
    ({"weight_dtype": "fp8_e4m3", "sk_clusterk": 7}, "needs sk_clusterk = 0"),
    ({"weight_dtype": "fp8_e4m3", "sk_clusterk": 2}, "needs sk_clusterk = 0"),
])
def test_weight_dtype_refusals(cfg, msg):
    rc, _ = _model_info({"model": "llama-3-8b", **cfg})
    assert rc == _lib.OA_ERR_BAD_REQUEST
    assert msg in _lib.last_error()


def test_bf16_options_still_accepted_with_tp_and_clusterk():
    assert _model_info({"model": "llama-3-8b", "tp": 2, "sk_clusterk": 7})[0] == 0
    assert _model_info({"model": "llama-3-8b", "weight_dtype": "bf16", "tp": 2, "sk_clusterk": 7})[0] == 0


def _np_row_rule(x):
    """independent restatement: s = 2^k, k the smallest integer with amax <= 448 * 2^k (clamped to >= -126); q = e4m3(x / s) via torch"""
    x = np.asarray(x, np.float32)
    amax = float(np.abs(x).max()) if x.size else 0.0
    if amax == 0.0:
        k = 0
    else:
        k = int(np.ceil(np.log2(amax / 448.0)))
        while amax > 448.0 * 2.0 ** k:
            k += 1
        while k > -126 and amax <= 448.0 * 2.0 ** (k - 1):
            k -= 1
        k = max(k, -126)
    s = np.float32(2.0 ** k)
    q = torch.from_numpy(x / s).to(torch.float8_e4m3fn)
    return q.view(torch.uint8).numpy(), float(s), q.float().numpy() * s


def test_row_rule_matches_numpy():
    rng = np.random.default_rng(11)
    rows = [np.zeros(64, np.float32),                                          # all zero: s = 1
            np.array([0, 0, 448, -0.0, 3], np.float32),                        # tie: amax = 448 * 2^0 exactly -> s = 1
            np.array([448.0001, 1], np.float32),                               # just above -> s = 2
            np.array([896, -896, 0.5], np.float32), np.array([897, 1], np.float32),
            np.array([7.0, -1.75 * 2.0 ** -20], np.float32),                   # 1.75 mantissa boundary
            np.array([1e-40, -3e-41, 0], np.float32),                          # subnormal amax -> clamped 2^-126
            np.array([3.0e38, -1.0], np.float32),                              # huge
            np.array([2.0 ** -120, 2.0 ** -121], np.float32)]
    rows += [(rng.standard_normal(300) * 10.0 ** rng.uniform(-6, 6)).astype(np.float32) for _ in range(40)]
    # every bf16 magnitude as the row maximum
    mags = O._np_bf16_to_f32(np.arange(0x0001, 0x7f80, 97, dtype=np.uint32).astype(np.uint16))
    rows += [np.array([m, m / 3, -m / 7], np.float32) for m in mags]
    for x in rows:
        q, s, d = w8_row(x)
        rq, rs, rd = _np_row_rule(x)
        assert s == rs, (x[:3], s, rs)
        assert np.array_equal(q, rq), x[:3]
        assert np.array_equal(d, rd.astype(np.float32))
        assert float(np.abs(x).max()) <= 448.0 * s and (s == 2.0 ** -126 or float(np.abs(x).max()) > 224.0 * s or s == 1.0)


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-qwen", "tiny-llama-d128"])
def test_mode3_switched_off_is_mode1_bit_for_bit(name):
    spec = O.PRESETS[name]
    toks = np.random.default_rng(5).integers(0, spec.vocab, size=40).astype(np.int32)
    ref = O.Oracle(spec, max_pos=64, mode=1)
    r1 = ref.forward(toks, all_logits=True); g1 = ref.generate(toks[:12], 6)
    ref.close()
    off = W8Oracle(spec, max_pos=64, w8=False)
    assert np.array_equal(off.forward(toks, all_logits=True), r1)
    off.close()
    off = W8Oracle(spec, max_pos=64, w8=False)
    g = off.generate(toks[:12], 6)
    off.close()
    assert np.array_equal(g[0], g1[0]) and np.array_equal(g[1], g1[1])
    # mode 2 (fp8 KV) with the switch off is mode 2
    m2 = Fp8Oracle(spec, max_pos=64)
    r2 = m2.forward(toks, all_logits=True)
    m2.close()
    off2 = W8Oracle(spec, max_pos=64, w8=False, kv_fp8=True)
    assert np.array_equal(off2.forward(toks, all_logits=True), r2)
    off2.close()


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-qwen"])
def test_mode3_quantises_the_projections(name):
    spec = O.PRESETS[name]
    toks = np.random.default_rng(6).integers(0, spec.vocab, size=48).astype(np.int32)
    ref = O.Oracle(spec, max_pos=64, mode=1)
    r1 = ref.forward(toks, all_logits=True)
    wq = ref.tensor_f32(0, "wq", (spec.n_heads * spec.head_dim, spec.hidden))
    ref.close()
    m3 = W8Oracle(spec, max_pos=64)
    r3 = m3.forward(toks, all_logits=True)
    # weights: e4m3(w / s_w) * s_w per row, which is a bf16 value
    got = m3.weight_f32(0, "wq", wq.shape)
    for n in range(0, wq.shape[0], 17):
        assert np.array_equal(got[n], _np_row_rule(wq[n])[2].astype(np.float32))
    assert np.array_equal(O._np_bf16_to_f32(O.f32_to_bf16_bits(got)), got)
    m3.close()
    d = np.abs(r3 - r1)
    assert 1e-3 < d.max() < 0.5, d.max()          # really quantised, by e4m3 rounding and not garbage
    # incremental decode is the same computation as the one-shot prefill (row-wise quantisation)
    m = W8Oracle(spec, max_pos=64)
    m.forward(toks[:40], all_logits=True)
    step = np.concatenate([m.forward(toks[i:i + 1], pos0=i) for i in range(40, 48)])
    m.close()
    assert np.abs(step - r3[40:]).max() < 1e-4


def _fake_quant_rows(t):
    """torch restatement of the row rule on the last dimension: x -> e4m3(x / s) * s"""
    amax = t.abs().amax(dim=-1, keepdim=True).double()
    k = torch.ceil(torch.log2(torch.clamp(amax, min=1e-300) / 448.0))
    k = torch.where(amax > 448.0 * torch.exp2(k), k + 1, k)
    k = torch.where(amax <= 448.0 * torch.exp2(k - 1), k - 1, k)
    k = torch.where(amax == 0, torch.zeros_like(k), torch.clamp(k, min=-126))
    s = torch.exp2(k).float()
    return (t / s).to(torch.float8_e4m3fn).float() * s


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-qwen"])
def test_mode0_w8a8_matches_a_torch_restatement(name):
    """mode 0 + W8A8 against HF transformers in fp32 with fake-quantised projection weights and inputs (forward pre-hooks)"""
    pytest.importorskip("transformers")
    from golden.gen_golden_hf import hf_model
    spec = O.PRESETS[name]
    base = O.Oracle(spec, max_pos=64, mode=0)
    model = hf_model(spec, base)
    base.close()
    names = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
    with torch.no_grad():
        for mn, mod in model.named_modules():
            if mn.split(".")[-1] in names:
                mod.weight.copy_(_fake_quant_rows(mod.weight))
                mod.register_forward_pre_hook(lambda _m, args: (_fake_quant_rows(args[0]),) + tuple(args[1:]))
        toks = np.random.default_rng(7).integers(0, spec.vocab, size=24).astype(np.int64)
        hf = model(torch.from_numpy(toks)[None]).logits[0].float().numpy()
    m3 = W8Oracle(spec, max_pos=64, mode=0)
    got = m3.forward(toks.astype(np.int32), all_logits=True)
    m3.close()
    err = float(np.abs(got - hf).max())
    assert err < 2e-4, err
