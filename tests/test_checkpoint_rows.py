"""The host half of the checkpoint loader (opsagent_b200/csrc/checkpoint.hpp) on the CPU: a C++ driver assembles every matrix a tensor-parallel
rank loads from a safetensors file, and the rows must equal numpy slicing of the oracle's tensors — q|k|v row shards, o / down column shards,
the 16-row gate/up interleave, bias shards, the vocab-parallel LM head — for BF16 / F16 / F32 checkpoints at every rank of tp = 1, 2, 4, 8
the preset supports.  F8_E4M3 projections: bytes and per-row / per-tensor scales in F32 / BF16 / F16, and every refusal's message."""
import json
import os
import struct
import subprocess

import numpy as np
import pytest

from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "opsagent_b200", "csrc")

# argv: checkpoint out_dir w8 tp hidden n_layers n_heads n_kv_heads head_dim ffn vocab tie_embeddings qkv_bias.  For every rank, every matrix
# the engine loads -> out_dir/r{rank}.{name}: bf16 rows (.u16), or e4m3 bytes (.u8) + row scales (.f32).  A refusal: "error: <message>", exit 3.
SRC = r'''
#include <cstdio>
#include <cstdlib>
#include "checkpoint.hpp"
using namespace oa;
static std::string out_dir;
template <class T> static void dump(int r, const std::string& name, const char* ext, const std::vector<T>& v) {
    FILE* f = std::fopen((out_dir + "/r" + std::to_string(r) + "." + name + ext).c_str(), "wb");
    std::fwrite(v.data(), sizeof(T), v.size(), f); std::fclose(f);
}
int main(int argc, char** argv) {
    if (argc != 14) return 2;
    out_dir = argv[2];
    const bool w8 = std::atoi(argv[3]); const int tp = std::atoi(argv[4]);
    ModelConfig c; c.hidden = std::atoi(argv[5]); c.n_layers = std::atoi(argv[6]); c.n_heads = std::atoi(argv[7]); c.n_kv_heads = std::atoi(argv[8]);
    c.head_dim = std::atoi(argv[9]); c.ffn = std::atoi(argv[10]); c.vocab = std::atoi(argv[11]); c.tie_embeddings = std::atoi(argv[12]); c.qkv_bias = std::atoi(argv[13]);
    try {
        SafeTensors st(argv[1]);
        std::vector<uint16_t> hb; std::vector<uint8_t> hq; std::vector<float> hs;
        for (int r = 0; r < tp; ++r) {
            const CkptShard s(st, c, tp, r);
            auto load = [&](const std::string& name, const CkptRows& m) { ckpt_bf16(st, m, hb); dump(r, name, ".u16", hb); };
            auto load_proj = [&](const std::string& name, const CkptRows& m) {
                if (!ckpt_is_f8(st, m, w8)) { load(name, m); return; }
                ckpt_f8(st, m, hq, hs); dump(r, name, ".u8", hq); dump(r, name, ".f32", hs);
            };
            load("embed", s.embed); load("norm", s.norm);
            if (!c.tie_embeddings) load("lm_head", s.lm_head);
            for (int l = 0; l < c.n_layers; ++l) {
                const CkptLayerRows& m = s.layers[l]; const std::string p = std::to_string(l) + ".";
                load_proj(p + "qkv", m.qkv); load_proj(p + "o", m.o); load_proj(p + "gu", m.gu); load_proj(p + "down", m.down);
                load(p + "ln1", m.ln1); load(p + "ln2", m.ln2);
                if (c.qkv_bias) load(p + "bqkv", m.bqkv);
            }
        }
    } catch (const std::exception& e) { std::printf("error: %s\n", e.what()); return 3; }
    return 0;
}
'''

PRESETS = ["tiny-llama", "tiny-qwen", "tiny-llama-tp", "tiny-qwen-tp4", "tiny-llama-tp8"]


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt_driver")
    src = d / "driver.cu"; src.write_text(SRC)
    exe = d / "driver"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    b = subprocess.run([nvcc, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, str(src), "-o", str(exe)],
                       capture_output=True, text=True, timeout=600)
    assert b.returncode == 0, b.stderr[-2000:]
    return str(exe)


def _run(exe, ckpt, out, spec, tp=1, w8=False, **override):
    dims = dict(hidden=spec.hidden, n_layers=spec.n_layers, n_heads=spec.n_heads, n_kv_heads=spec.n_kv_heads, head_dim=spec.head_dim, ffn=spec.ffn,
                vocab=spec.vocab, tie_embeddings=spec.tie_embeddings, qkv_bias=spec.qkv_bias)
    dims.update(override)
    os.makedirs(out, exist_ok=True)
    return subprocess.run([exe, str(ckpt), str(out), str(int(w8)), str(tp)] + [str(v) for v in dims.values()], capture_output=True, text=True, timeout=120)


def _tp_degrees(spec):
    """the tensor-parallel degrees the engine accepts for this preset"""
    return [t for t in (1, 2, 4, 8) if spec.n_kv_heads % t == 0 and spec.n_heads % t == 0 and spec.ffn % t == 0 and (spec.ffn // t) % 64 == 0
            and spec.vocab % t == 0 and (spec.vocab // t) % 8 == 0]


def _as_stored(bits, dtype):
    """bf16 bits of an oracle tensor after a round trip through a checkpoint of `dtype` (F16 rounds; BF16 / F32 are exact)"""
    if dtype != "F16":
        return bits
    return O.f32_to_bf16_bits(O._np_bf16_to_f32(bits).astype(np.float16).astype(np.float32))


def _expected(orc, dtype, tp, r):
    """name -> this rank's rows, by numpy slicing of the oracle's (logical, unsharded) tensors"""
    sp = orc.spec
    H, qd, kd, F, V = sp.hidden, sp.n_heads * sp.head_dim, sp.n_kv_heads * sp.head_dim, sp.ffn, sp.vocab
    ql, kl, Fl, Vl = qd // tp, kd // tp, F // tp, V // tp
    t = lambda l, kind, shape: _as_stored(orc.tensor(l, kind, shape), dtype)      # noqa: E731
    rows = lambda a, n: a[r * n:(r + 1) * n]                                        # noqa: E731
    embed = t(-1, 0, (V, H))
    out = {"embed": embed, "norm": t(-1, 1, (H,))}
    if not sp.tie_embeddings:
        out["lm_head"] = rows(t(-1, 2, (V, H)), Vl)
    for l in range(sp.n_layers):
        p = f"{l}."
        out[p + "qkv"] = np.concatenate([rows(t(l, "wq", (qd, H)), ql), rows(t(l, "wk", (kd, H)), kl), rows(t(l, "wv", (kd, H)), kl)])
        out[p + "o"] = t(l, "wo", (H, qd))[:, r * ql:(r + 1) * ql]
        g, u = rows(t(l, "wg", (F, H)), Fl), rows(t(l, "wu", (F, H)), Fl)
        out[p + "gu"] = np.stack([g.reshape(-1, 16, H), u.reshape(-1, 16, H)], axis=1).reshape(2 * Fl, H)       # 16 gate rows, 16 up rows, ...
        out[p + "down"] = t(l, "wd", (H, F))[:, r * Fl:(r + 1) * Fl]
        out[p + "ln1"], out[p + "ln2"] = t(l, "ln1", (H,)), t(l, "ln2", (H,))
        if sp.qkv_bias:
            out[p + "bqkv"] = np.concatenate([rows(t(l, "bq", (qd,)), ql), rows(t(l, "bk", (kd,)), kl), rows(t(l, "bv", (kd,)), kl)])
    return out


@pytest.mark.parametrize("dtype", ["BF16", "F16", "F32"])
@pytest.mark.parametrize("name", PRESETS)
def test_checkpoint_shards_equal_numpy_slicing(driver, name, dtype, tmp_path):
    spec = O.PRESETS[name]
    orc = O.Oracle(spec, max_pos=64, mode=1)
    ckpt = tmp_path / "model.safetensors"
    O.write_safetensors(orc, str(ckpt), dtype)
    degrees = _tp_degrees(spec)
    assert degrees[0] == 1 and (len(degrees) > 1 or name == "tiny-qwen")
    for tp in degrees:
        out = tmp_path / f"tp{tp}"
        res = _run(driver, ckpt, out, spec, tp=tp)
        assert res.returncode == 0, res.stdout + res.stderr
        for r in range(tp):
            for key, want in _expected(orc, dtype, tp, r).items():
                got = np.fromfile(out / f"r{r}.{key}.u16", dtype=np.uint16)
                assert np.array_equal(got, want.reshape(-1)), (name, dtype, tp, r, key)
    orc.close()


# ------------------------------------------------------------------------------------------------ F8_E4M3 projections
PROJ = {"wq": "self_attn.q_proj", "wk": "self_attn.k_proj", "wv": "self_attn.v_proj", "wo": "self_attn.o_proj", "wg": "mlp.gate_proj",
        "wu": "mlp.up_proj", "wd": "mlp.down_proj"}
# every scale dtype with every scale shape: per row [N, 1] / [N], per tensor [] / [1]
STYLES = [(dt, shape) for dt in ("F32", "BF16", "F16") for shape in ("row2", "row1", "tensor0", "tensor1")]


def _read(path):
    raw = open(path, "rb").read()
    n = struct.unpack("<Q", raw[:8])[0]
    hdr, body = json.loads(raw[8:8 + n]), raw[8 + n:]
    return {k: [m["dtype"], m["shape"], body[m["data_offsets"][0]:m["data_offsets"][1]]] for k, m in hdr.items() if k != "__metadata__"}


def _write(path, items):
    header, blobs, off = {"__metadata__": {"format": "pt"}}, [], 0
    for name, (dt, shape, raw) in items.items():
        header[name] = {"dtype": dt, "shape": list(shape), "data_offsets": [off, off + len(raw)]}
        blobs.append(raw); off += len(raw)
    hj = json.dumps(header, separators=(",", ":")).encode(); hj += b" " * ((8 - len(hj) % 8) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(hj))); f.write(hj)
        for b in blobs:
            f.write(b)


def _scale_raw(s, dt):
    if dt == "F32":
        return s.astype(np.float32).tobytes()
    if dt == "BF16":
        return O.f32_to_bf16_bits(s).tobytes()
    return s.astype(np.float16).tobytes()


def _fp8_items(orc, rng, tmp_dir):
    """the oracle's checkpoint with every projection as F8_E4M3 bytes + a `_scale` tensor (styles cycled over the matrices).
    -> (items, {(layer, kind): (bytes [N, K], fp32 scale of each row)})"""
    sp = orc.spec
    H, qd, kd, F = sp.hidden, sp.n_heads * sp.head_dim, sp.n_kv_heads * sp.head_dim, sp.ffn
    shapes = {"wq": (qd, H), "wk": (kd, H), "wv": (kd, H), "wo": (H, qd), "wg": (F, H), "wu": (F, H), "wd": (H, F)}
    tmp = str(tmp_dir / "bf16.safetensors")
    O.write_safetensors(orc, tmp)
    items, want = _read(tmp), {}
    for l in range(sp.n_layers):
        for i, (kind, shp) in enumerate(shapes.items()):
            dt, style = STYLES[(i + 7 * l) % len(STYLES)]
            nm = f"model.layers.{l}.{PROJ[kind]}.weight"
            qb = rng.integers(0, 256, size=shp, dtype=np.uint8)
            qb[(qb & 0x7F) == 0x7F] = 0                         # no e4m3 NaN codes
            s = rng.uniform(1e-3, 1e-2, size=shp[0] if style.startswith("row") else 1).astype(np.float32)
            s = np.frombuffer(_scale_raw(s, dt), {"F32": np.float32, "BF16": np.uint16, "F16": np.float16}[dt])
            s = O._np_bf16_to_f32(s) if dt == "BF16" else s.astype(np.float32)
            sshape = {"row2": [shp[0], 1], "row1": [shp[0]], "tensor0": [], "tensor1": [1]}[style]
            items[nm] = ["F8_E4M3", list(shp), qb.tobytes()]
            items[nm + "_scale"] = [dt, sshape, _scale_raw(s, dt)]
            items[nm.replace(".weight", ".input_scale")] = ["F32", [], np.float32(0.5).tobytes()]      # not read (dynamic activation scales)
            want[(l, kind)] = (qb, np.broadcast_to(s, (shp[0],)))
    return items, want


def test_fp8_checkpoint_rows_and_scales(driver, tmp_path):
    spec = O.PRESETS["tiny-llama"]
    orc = O.Oracle(spec, max_pos=64, mode=1)
    items, want = _fp8_items(orc, np.random.default_rng(5), tmp_path)
    ckpt = tmp_path / "fp8.safetensors"
    _write(ckpt, items)
    res = _run(driver, ckpt, tmp_path / "out", spec, w8=True)
    assert res.returncode == 0, res.stdout + res.stderr
    F = spec.ffn
    for l in range(spec.n_layers):
        w = {k: want[(l, k)] for k in PROJ}
        exp = {"qkv": [w["wq"], w["wk"], w["wv"]], "o": [w["wo"]], "down": [w["wd"]]}
        for key, parts in exp.items():
            qb, sc = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
            assert np.array_equal(np.fromfile(tmp_path / "out" / f"r0.{l}.{key}.u8", np.uint8), qb.reshape(-1)), (l, key)
            assert np.array_equal(np.fromfile(tmp_path / "out" / f"r0.{l}.{key}.f32", np.float32), sc), (l, key)
        order = np.stack([np.arange(F).reshape(-1, 16), F + np.arange(F).reshape(-1, 16)], axis=1).reshape(-1)     # gate/up interleave
        qb, sc = np.concatenate([w["wg"][0], w["wu"][0]])[order], np.concatenate([w["wg"][1], w["wu"][1]])[order]
        assert np.array_equal(np.fromfile(tmp_path / "out" / f"r0.{l}.gu.u8", np.uint8), qb.reshape(-1)), l
        assert np.array_equal(np.fromfile(tmp_path / "out" / f"r0.{l}.gu.f32", np.float32), sc), l
    # the bf16 tensors of the same file load as they do from a bf16 checkpoint
    exp = _expected(orc, "BF16", 1, 0)
    for key in ("embed", "norm", "lm_head", "0.ln1", "1.ln2"):
        assert np.array_equal(np.fromfile(tmp_path / "out" / f"r0.{key}.u16", np.uint16), exp[key].reshape(-1)), key

    # refusals, each with a message naming the problem
    H, V = spec.hidden, spec.vocab
    kd = spec.n_kv_heads * spec.head_dim
    q0 = "model.layers.0.self_attn.q_proj.weight"
    bad = {
        "missing scale": ({q0 + "_scale": None}, ["q_proj.weight_scale", "is missing"]),
        "bad scale shape": ({q0 + "_scale": ["F32", [3], np.ones(3, np.float32).tobytes()]}, ["q_proj.weight_scale", "must have shape"]),
        "negative scale": ({q0 + "_scale": ["F32", [], np.float32(-1).tobytes()]}, ["q_proj.weight_scale", "must be finite and > 0"]),
        "zero scale": ({q0 + "_scale": ["F16", [1], np.float16(0).tobytes()]}, ["q_proj.weight_scale", "must be finite and > 0"]),
        "nan scale": ({q0 + "_scale": ["BF16", [1], np.uint16(0x7FC0).tobytes()]}, ["q_proj.weight_scale", "must be finite and > 0"]),
        "int scale": ({q0 + "_scale": ["I32", [], np.int32(1).tobytes()]}, ["q_proj.weight_scale", "unsupported dtype"]),
        "fp8 embedding": ({"model.embed_tokens.weight": ["F8_E4M3", [V, H], bytes(V * H)]}, ["embed_tokens", "unsupported dtype F8_E4M3"]),
        "mixed q/k": ({"model.layers.1.self_attn.k_proj.weight": ["BF16", [kd, H], bytes(2 * kd * H)]}, ["must all be F8_E4M3 or none"]),
    }
    for why, (change, msgs) in bad.items():
        it = dict(items)
        for k, v in change.items():
            if v is None:
                del it[k]
            else:
                it[k] = v
        p = tmp_path / f"bad_{why.replace(' ', '_').replace('/', '_')}.safetensors"
        _write(p, it)
        res = _run(driver, p, tmp_path / "bad", spec, w8=True)
        assert res.returncode == 3 and all(m in res.stdout for m in msgs), (why, res.stdout, res.stderr)
    res = _run(driver, ckpt, tmp_path / "bad", spec, w8=False)          # F8 projections under weight_dtype bf16
    assert res.returncode == 3 and "_proj.weight is F8_E4M3" in res.stdout and "weight_dtype fp8_e4m3" in res.stdout, res.stdout
    res = _run(driver, ckpt, tmp_path / "bad", spec, w8=True, ffn=2 * spec.ffn)          # a checkpoint of another configuration
    assert res.returncode == 3 and "has shape" in res.stdout, res.stdout
    orc.close()
