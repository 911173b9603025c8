"""Mode 2 of the CPU oracle for the fp8 (e4m3) KV cache (tests/kv_fp8_oracle.c): oracle/llama_ref.c compiled unchanged, with the copies
into the KV cache quantised to e4m3(x / s) * s.  TEST INFRASTRUCTURE ONLY.

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


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="oa_kv_fp8_oracle_"), "libkvfp8oracle.so")
        subprocess.run(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-fvisibility=hidden",
                        "-Wall", "-Wno-unused-function", "-shared", "-o", out, os.path.join(_HERE, "kv_fp8_oracle.c"), "-lm"], check=True)
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")
        L = C.CDLL(out)
        L.oa_ref2_create.restype = C.c_void_p
        L.oa_ref2_create.argtypes = [C.POINTER(O.RefConfig), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.oa_ref2_destroy.argtypes = [C.c_void_p]
        L.oa_ref_forward.restype = C.c_int
        L.oa_ref_forward.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.oa_ref_generate.restype = C.c_int32
        L.oa_ref_generate.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oa_ref_e4m3.restype = C.c_uint8
        L.oa_ref_e4m3.argtypes = [C.c_float]
        L.oa_ref_e4m3_to_f32.restype = C.c_float
        L.oa_ref_e4m3_to_f32.argtypes = [C.c_uint8]
        L.oa_ref_set_threads.argtypes = [C.c_int32]
        L.oa_ref_set_threads(O.default_threads())
        _LIB = L
    return _LIB


def e4m3(x) -> np.ndarray:
    """the oracle's fp32 -> e4m3 byte (round to nearest even, saturating to +-448)"""
    f = lib().oa_ref_e4m3
    return np.array([f(float(v)) for v in np.asarray(x, np.float32).ravel()], np.uint8).reshape(np.shape(x))


def e4m3_to_f32(b) -> np.ndarray:
    f = lib().oa_ref_e4m3_to_f32
    return np.array([f(int(v)) for v in np.asarray(b, np.uint8).ravel()], np.float32).reshape(np.shape(b))


class Fp8Oracle(O.Oracle):
    """O.Oracle in mode 2: k_scale / v_scale are per-layer lists (None: 1.0).  forward() and generate() as in O.Oracle."""

    def __init__(self, spec: "O.ModelSpec", max_pos: int = 512, n_slots: int = 1, k_scale=None, v_scale=None):
        self.spec, self.max_pos, self.n_slots, self.mode = spec, max_pos, n_slots, 2
        self._cfg = spec.to_c()
        ks = None if k_scale is None else np.ascontiguousarray(k_scale, np.float32)
        vs = None if v_scale is None else np.ascontiguousarray(v_scale, np.float32)
        self._h = lib().oa_ref2_create(C.byref(self._cfg), max_pos, n_slots, ks.ctypes.data if ks is not None else None,
                                       vs.ctypes.data if vs is not None else None)
        if not self._h:
            raise MemoryError("oa_ref2_create failed")

    def close(self):
        if self._h:
            lib().oa_ref2_destroy(self._h)
            self._h = None

    def tensor(self, layer, kind, shape):
        raise NotImplementedError("use an O.Oracle of the same spec for the weights")

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
