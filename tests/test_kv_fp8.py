"""fp8 (e4m3) KV cache, CPU side: the e4m3 arithmetic of the oracle's mode 2 (tests/kv_fp8_oracle.c), the kv_cache_dtype option as the host
parses it, and mode 2 itself, which the GPU tests hold the engine to."""
import ctypes as C
import json

import numpy as np
import pytest

from kv_fp8_ref import Fp8Oracle, e4m3, e4m3_to_f32
from opsagent_b200 import _lib
from oracle import oracle as O

torch = pytest.importorskip("torch")


def _all_bf16_as_f32():
    return O._np_bf16_to_f32(np.arange(1 << 16, dtype=np.uint32).astype(np.uint16))


def test_oracle_e4m3_matches_torch_for_every_bf16_value():
    x = _all_bf16_as_f32()
    fin = np.isfinite(x)
    got = e4m3(x[fin])
    ref = torch.from_numpy(x[fin]).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    small = np.abs(x[fin]) < 464          # torch rounds these like the hardware; beyond, torch gives NaN and satfinite gives +-448
    assert np.array_equal(got[small], ref[small])
    big = x[fin][~small]
    assert len(big) > 0 and np.array_equal(got[~small], np.where(big < 0, 0xFE, 0x7E).astype(np.uint8))
    assert np.isin(got, [0x7F, 0xFF]).sum() == 0          # never a NaN code


def test_oracle_e4m3_decode_matches_torch():
    b = np.arange(256, dtype=np.uint8)
    ref = torch.from_numpy(b).view(torch.float8_e4m3fn).float().numpy()
    got = e4m3_to_f32(b)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan], ref[~nan])
    assert got[0] == 0.0                  # the zero-filled pool reads as +0


def _q(x, s):
    inv = np.float32(1.0) / np.float32(s)
    return e4m3_to_f32(e4m3(np.asarray(x, np.float32) * inv)) * np.float32(s)


def test_scale_algebra():
    rng = np.random.default_rng(3)
    x = (rng.standard_normal(4096) * 3).astype(np.float32)
    # a power-of-two scale only shifts the exponent: same relative grid, as long as nothing saturates or goes subnormal
    for s in (0.25, 2.0, 4.0):
        y = x[(np.abs(x / s) < 400) & (np.abs(x / s) > 2.0 ** -6)]
        assert np.array_equal(_q(y, s), _q(y / np.float32(s), 1.0) * np.float32(s))
    # one rounding: at most half an e4m3 step (2^-4 relative) for normal values
    y = x[np.abs(x) > 2.0 ** -6]
    assert (np.abs(_q(y, 1.0) - y) <= np.abs(y) * 2.0 ** -4 + 1e-9).all()
    # a scale moves the saturation point: x = 960 with s = 4 is stored exactly as 240; with s = 1 it saturates at 448
    assert _q(960, 4.0) == 960 and _q(960, 1.0) == 448


def _model_info(cfg):
    L = _lib.load()
    buf = C.create_string_buffer(2048)
    rc = L.oa_host_model_info(json.dumps(cfg).encode(), buf, 2048)
    return rc, (json.loads(buf.value.decode()) if rc == 0 else None)


@pytest.mark.parametrize("name", ["llama-3-8b", "llama-3.2-1b", "tiny-llama"])
def test_model_info_reports_the_fp8_cache(name):
    cfg = {"model": name} if name in ("llama-3-8b", "llama-3.2-1b") else O.PRESETS[name].engine_json()
    rc, base = _model_info(cfg)
    assert rc == 0 and "kv_cache_dtype" not in base            # default output as before
    rc, bf = _model_info({**cfg, "kv_cache_dtype": "bf16"})
    assert rc == 0 and bf == base
    rc, f8 = _model_info({**cfg, "kv_cache_dtype": "fp8_e4m3"})
    assert rc == 0 and f8["kv_cache_dtype"] == "fp8_e4m3"
    assert f8["kv_bytes_per_token"] * 2 == base["kv_bytes_per_token"]
    if name == "llama-3-8b":
        assert f8["kv_bytes_per_token"] == 2 * 32 * 8 * 128         # K and V, 32 layers, 8 kv heads x 128 dims, one byte each


@pytest.mark.parametrize("bad", ["fp8", "e4m3", "FP8_E4M3", "fp16", ""])
def test_unknown_kv_cache_dtype_is_refused(bad):
    rc, _ = _model_info({"model": "llama-3-8b", "kv_cache_dtype": bad})
    assert rc == _lib.OA_ERR_BAD_REQUEST


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-qwen", "tiny-llama-d128"])
def test_oracle_mode2_quantizes_the_cache(name):
    spec = O.PRESETS[name]
    rng = np.random.default_rng(5)
    toks = rng.integers(0, spec.vocab, size=70).astype(np.int32)
    orc1 = O.Oracle(spec, max_pos=128, mode=1)
    ref1 = orc1.forward(toks, all_logits=True)
    orc1.close()
    m2 = Fp8Oracle(spec, max_pos=128)
    q1 = m2.forward(toks, all_logits=True)
    m2.close()
    # position 0 attends to itself only: softmax of one score is 1, so the output is its quantised v row and logits still move
    d = np.abs(q1 - ref1)
    assert d[0].max() > 1e-3 and d.max() > 3e-2, (d[0].max(), d.max())          # unit scales: the cache really is quantised
    assert d.max() < 1.0                                                          # ... by one e4m3 rounding, not garbage
    # a power-of-two scale on every layer moves only values that were subnormal or saturated: close to unit scales
    s = [2.0] * spec.n_layers
    m2s = Fp8Oracle(spec, max_pos=128, k_scale=s, v_scale=s)
    qs = m2s.forward(toks, all_logits=True)
    m2s.close()
    assert np.abs(qs - q1).max() < np.abs(q1 - ref1).max()
    # incremental decode through the quantised cache: the same computation as the one-shot prefill, token by token
    m = Fp8Oracle(spec, max_pos=128)
    m.forward(toks[:64], all_logits=True)
    step = np.concatenate([m.forward(toks[i:i + 1], pos0=i) for i in range(64, 70)])
    m.close()
    assert np.abs(step - q1[64:]).max() < 1e-4
