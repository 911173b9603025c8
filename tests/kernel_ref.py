"""Shared checking helpers of the kernel-level GPU tests (tests/test_decode_kernels_gpu.py, tests/test_prefill_kernels_gpu.py): bf16 ulps,
the "within 1 ulp of the fp64 reference, with an exact-match floor" check, bitwise equality, the engine's e4m3 row quantiser and the
projection tolerances.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import torch

BF16, FP8 = torch.bfloat16, torch.float8_e4m3fn

# Bounds.  Every output is within 1 bf16 ulp of its reference, where a near-zero reference (a sum that cancels) takes the
# projection's accumulation error instead.  The tensor core's fp32 accumulation truncates, so its error grows linearly with K: measured
# up to 2^-29 K of the product's rms (3e-5 at K = 14336), bounded here by 2^-26 K.  With e4m3 operands it adds the 128 products of a
# k block with about 14 mantissa bits (5e-4 of the largest output, tests/test_w8_fp8_gpu.py).
ACC_TOL_BF16_PER_K, ACC_TOL_FP8 = 2.0 ** -26, 5e-4
# Fraction of outputs exactly equal to the rounded fp64 reference.  Measured on an H100 SXM (132 SMs, default power limit), smallest over
# all shapes and variants of tests/test_decode_kernels_gpu.py: bf16 operands 0.9917 (gate/up at Llama-3-70B), 0.9924 (x at K <= 16384),
# 0.9922 (v), > 0.997 (xn, q, k, the fp8 K / V bytes); the down projections of Qwen2.5-32B and Llama-3-70B (K = 27648, 28672) 0.9853 and
# 0.9838 (x: the truncation error grows with K); e4m3 operands 0.883 (gate/up), 0.925 (v), 0.944 (x), 0.949 (q), > 0.99 (the fp8 K / V
# bytes, xn).
MIN_EQUAL, MIN_EQUAL_LONG_K = 0.99, 0.98
MIN_EQUAL_FP8 = 0.85

MATCH = {}                   # smallest measured exact-match fraction per check, printed by each test (pytest -s)


def dev():
    return torch.device("cuda:0")


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def quant(L, x):
    """e4m3 rows + fp32 row scales through the engine's quantiser, and their fp64 value e4m3 * scale"""
    R, Cc = x.shape
    q = torch.empty(R, Cc, dtype=torch.uint8, device=x.device); s = torch.empty(R, dtype=torch.float32, device=x.device)
    assert L.oa_k_quant_rows_e4m3(ptr(x), ptr(q), ptr(s), R, Cc, None) == 0
    return q, s, q.view(FP8).double() * s.double()[:, None]


def ulp(a):
    """bf16 ulp of |a| (fp64): 2^(exponent - 7)"""
    return torch.exp2(torch.floor(torch.log2(a.abs().clamp_min(2.0 ** -126))) - 7)


def check_bf16(got, ref, what, lo=None, hi=None, abs_tol=0.0, min_equal=MIN_EQUAL):
    """bf16 `got` within 1 ulp (or abs_tol) of the fp64 reference interval [lo, hi] (default: the point ref); at least min_equal of it
    equal to bf16(ref).  Returns that fraction."""
    lo = ref if lo is None else lo
    hi = ref if hi is None else hi
    g = got.double()
    tol = torch.maximum(ulp(torch.maximum(lo.abs(), hi.abs())), torch.full_like(lo, abs_tol))
    over = (g - torch.minimum(torch.maximum(g, lo), hi)).abs() - tol
    bad = ~(over <= 0)                                     # NaN counts as bad
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} outputs beyond 1 bf16 ulp; e.g. flat index {i}: kernel "
                             f"{g.flatten()[i].item()!r}, reference [{lo.flatten()[i].item()!r}, {hi.flatten()[i].item()!r}]")
    frac = (got == ref.to(BF16)).double().mean().item()
    key = what.split(":")[0]
    MATCH[key] = min(MATCH.get(key, 1.0), frac)
    assert frac >= min_equal, f"{what}: only {frac:.5f} of the outputs equal the rounded reference"
    return frac


def same(a, b):
    """bitwise equality (NaN sentinels included)"""
    return torch.equal(a.view(torch.int16), b.view(torch.int16)) if a.dtype == BF16 else torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def report(name):
    print(f"\n{name} exact-match fractions (min): " + ", ".join(f"{k} {v:.5f}" for k, v in sorted(MATCH.items())))
    MATCH.clear()
