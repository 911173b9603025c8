"""Mode 3 of the CPU oracle for fp8 (e4m3) projection weights (tests/w8_fp8_oracle.c): oracle/llama_ref.c compiled unchanged, with the seven
per-layer projections run as W8A8 (row-rule scales on weights and on every input row).  TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a temporary directory (the source tree may be read-only), with oracle/Makefile's flags."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
KINDS = {"wq": 0, "wk": 1, "wv": 2, "wo": 3, "wg": 4, "wu": 5, "wd": 6}


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="oa_w8_fp8_oracle_"), "libw8fp8oracle.so")
        subprocess.run(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-fvisibility=hidden",
                        "-Wall", "-Wno-unused-function", "-shared", "-o", out, os.path.join(_HERE, "w8_fp8_oracle.c"), "-lm"], check=True)
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")
        L = C.CDLL(out)
        vp, i32 = C.c_void_p, C.c_int32
        L.oa_ref_create.restype = vp
        L.oa_ref_create.argtypes = [C.POINTER(O.RefConfig), i32, i32, i32]
        L.oa_ref_destroy.argtypes = [vp]
        L.oa_ref2_create.restype = vp
        L.oa_ref2_create.argtypes = [C.POINTER(O.RefConfig), i32, i32, vp, vp]
        L.oa_ref2_destroy.argtypes = [vp]
        L.oa_ref3_enable.restype = C.c_int
        L.oa_ref3_enable.argtypes = [vp]
        L.oa_ref3_disable.argtypes = [vp]
        L.oa_ref3_set_weight.restype = C.c_int
        L.oa_ref3_set_weight.argtypes = [vp, i32, i32, vp, vp]
        L.oa_ref3_get_weight.restype = C.c_int
        L.oa_ref3_get_weight.argtypes = [vp, i32, i32, vp]
        L.oa_ref_tensor.restype = vp
        L.oa_ref_tensor.argtypes = [vp, i32, i32]
        L.oa_ref_forward.restype = C.c_int
        L.oa_ref_forward.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp]
        L.oa_ref_generate.restype = i32
        L.oa_ref_generate.argtypes = [vp, i32, vp, i32, i32, vp, i32, vp, vp, vp]
        L.oa_ref_w8_scale.restype = C.c_float
        L.oa_ref_w8_scale.argtypes = [C.c_float]
        L.oa_ref_w8_row.restype = C.c_float
        L.oa_ref_w8_row.argtypes = [vp, C.c_int, vp, vp]
        L.oa_ref_set_threads.argtypes = [i32]
        L.oa_ref_set_threads(O.default_threads())
        _LIB = L
    return _LIB


def w8_row(x) -> tuple[np.ndarray, float, np.ndarray]:
    """the oracle's row rule on one fp32 row: (e4m3 bytes, scale, dequantised row)"""
    x = np.ascontiguousarray(x, np.float32)
    q = np.empty(x.shape, np.uint8); d = np.empty(x.shape, np.float32)
    s = lib().oa_ref_w8_row(x.ctypes.data, len(x), q.ctypes.data, d.ctypes.data)
    return q, float(s), d


class W8Oracle(O.Oracle):
    """O.Oracle in mode 3: mode (0 or 1) plus W8A8 projections when w8; kv_fp8 adds mode 2's e4m3 KV cache (mode 1 only).
    forward() and generate() as in O.Oracle; set_weight() replaces one projection by e4m3 bytes and per-row scales."""

    def __init__(self, spec: "O.ModelSpec", max_pos: int = 512, n_slots: int = 1, mode: int = 1, w8: bool = True, kv_fp8: bool = False,
                 k_scale=None, v_scale=None):
        self.spec, self.max_pos, self.n_slots, self.mode = spec, max_pos, n_slots, mode
        self._cfg = spec.to_c()
        L = lib()
        if kv_fp8:
            assert mode == 1, "the fp8 KV cache oracle is mode 1 based"
            ks = None if k_scale is None else np.ascontiguousarray(k_scale, np.float32)
            vs = None if v_scale is None else np.ascontiguousarray(v_scale, np.float32)
            self._h = L.oa_ref2_create(C.byref(self._cfg), max_pos, n_slots, ks.ctypes.data if ks is not None else None,
                                       vs.ctypes.data if vs is not None else None)
        else:
            self._h = L.oa_ref_create(C.byref(self._cfg), max_pos, n_slots, mode)
        self._kv = kv_fp8
        if not self._h:
            raise MemoryError("oracle create failed")
        if w8 and L.oa_ref3_enable(self._h) != 0:
            raise MemoryError("oa_ref3_enable failed")

    def close(self):
        if self._h:
            L = lib()
            L.oa_ref3_disable(self._h)
            (L.oa_ref2_destroy if self._kv else L.oa_ref_destroy)(self._h)
            self._h = None

    def tensor(self, layer: int, kind, shape) -> np.ndarray:
        k = self.KINDS[kind] if isinstance(kind, str) else kind
        p = lib().oa_ref_tensor(self._h, layer, k)
        n = int(np.prod(shape))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint16)), (n,)).reshape(shape).copy()

    def weight_f32(self, layer: int, kind: str, shape) -> np.ndarray:
        out = np.empty(shape, np.float32)
        assert lib().oa_ref3_get_weight(self._h, layer, KINDS[kind], out.ctypes.data) == 0
        return out

    def set_weight(self, layer: int, kind: str, q: np.ndarray, s: np.ndarray) -> None:
        q = np.ascontiguousarray(q, np.uint8); s = np.ascontiguousarray(s, np.float32)
        assert lib().oa_ref3_set_weight(self._h, layer, KINDS[kind], q.ctypes.data, s.ctypes.data) == 0

    def forward(self, tokens, pos0: int = 0, slot: int = 0, all_logits: bool = False, want_hidden: bool = False):
        toks = np.ascontiguousarray(tokens, dtype=np.int32)
        logits = np.empty((len(toks) if all_logits else 1, self.spec.vocab), dtype=np.float32)
        if lib().oa_ref_forward(self._h, slot, toks.ctypes.data, len(toks), pos0, int(all_logits), logits.ctypes.data, None) != 0:
            raise ValueError("oa_ref_forward: bad slot or position")
        return logits

    def generate(self, prompt, max_new: int, eos=(), slot: int = 0):
        p = np.ascontiguousarray(prompt, dtype=np.int32)
        out = np.empty((max_new,), np.int32); mar = np.empty((max_new,), np.float32); fl = np.empty((self.spec.vocab,), np.float32)
        e = np.ascontiguousarray(list(eos), dtype=np.int32)
        n = lib().oa_ref_generate(self._h, slot, p.ctypes.data, len(p), max_new, e.ctypes.data if len(e) else None, len(e),
                                  out.ctypes.data, mar.ctypes.data, fl.ctypes.data)
        if n < 0:
            raise ValueError("oa_ref_generate failed")
        return out[:n].copy(), mar[:max(n, 1)].copy(), fl
