"""The decode step's finishing kernels at the single-GPU presets' decode shapes (pytest -m gpu): the o / down finish (residual + RMSNorm),
gate/up + SwiGLU, qkv + bias + RoPE + paged-KV write, the prefill KV writer, decode attention with the in-kernel merge and the LM head's
grammar-masked arg-max, each through the C entry point that launches it as DeviceModel::forward does, against an fp64 reference of the op
computed from the kernel's inputs and rounded to bf16 where the kernel rounds."""
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from opsagent_b200 import _lib  # noqa: E402
from kernel_ref import (ACC_TOL_BF16_PER_K, ACC_TOL_FP8, BF16, FP8, MATCH, MIN_EQUAL, MIN_EQUAL_FP8, MIN_EQUAL_LONG_K,  # noqa: E402
                        check_bf16, dev, ptr, quant, report, same, ulp)

BF16_NAN = 0x7FC0            # output sentinel: rows the kernel must not write keep these bits
KV_FILL_BF16 = 0x7F7F        # bf16 KV sentinel (a finite value no writer produces), fp8: 0x7F (an e4m3 NaN code no writer produces)
EPS = 1e-5
MAXM = 256                   # operand rows: every M below takes the first M rows, so one fp64 product serves all of them
MS = [1, 5, 64, 127, 128]
CLUSTERS = [2, 3, 4, 8]
MAX_POS = 16384              # positions beyond 8192

# name: (hidden, n_heads, n_kv, head_dim, ffn, qkv bias) of the single-GPU presets (csrc/config.hpp)
PRESETS = {
    "llama-3.2-1b": (2048, 32, 8, 64, 8192, False),
    "llama-3-8b": (4096, 32, 8, 128, 14336, False),
    "qwen2.5-32b": (5120, 40, 8, 128, 27648, True),
    "llama-3-70b": (8192, 64, 8, 128, 28672, False),
}
# one tensor-parallel rank's column-parallel layout (its heads and its ffn shard; hidden stays whole): the same qkv and gate/up kernels at
# shapes the single-GPU presets never make.  Not in PRESETS: the fused o / down finishers never run under tensor parallelism.
TP_RANKS = {
    "qwen2.5-32b/tp4": (5120, 10, 2, 128, 6912, True),
    "llama-3-70b/tp8": (8192, 8, 1, 128, 3584, False),
}
LAYOUTS = {**PRESETS, **TP_RANKS}

# Bounds and exact-match floors: tests/kernel_ref.py (measured on an H100 SXM, 132 SMs, default power limit).  The whole file runs in about
# 30 s on that GPU.


@pytest.fixture(scope="module")
def L():
    return _lib.load()


@pytest.fixture(autouse=True)
def _fresh_match_record():
    MATCH.clear()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gen(seed):
    return torch.Generator(device=dev()).manual_seed(seed)


# ------------------------------------------------------------------------------------------------ operands
class Proj:
    """One decode projection of a preset: A [MAXM, K] and B [N, K] in bf16 and as quantised e4m3 rows, and their fp64 products [MAXM, N]"""

    def __init__(self, L, N, K, seed):
        self.N, self.K = N, K
        g = gen(seed)
        self.A = torch.randn(MAXM, K, device=dev(), generator=g).to(BF16)
        self.B = (torch.randn(N, K, device=dev(), generator=g) * K ** -0.5).to(BF16)
        self.acc = self.A.double() @ self.B.double().T
        self.A8, self.sa, a8 = quant(L, self.A)
        self.B8, self.sb, b8 = quant(L, self.B)
        self.acc8 = a8 @ b8.T
        del a8, b8
        self.tol = ACC_TOL_BF16_PER_K * K * self.acc.pow(2).mean().sqrt().item()
        self.tol8 = ACC_TOL_FP8 * self.acc8.abs().max().item()
        self.min_equal = MIN_EQUAL if K <= 16384 else MIN_EQUAL_LONG_K

    def ops(self, fp8):
        return (self.A8, self.sa, self.B8, self.sb) if fp8 else (self.A, None, self.B, None)

    def product(self, fp8, M):
        return (self.acc8 if fp8 else self.acc)[:M], (self.tol8 if fp8 else self.tol)


_CACHE = {}


def proj(L, preset, kind, N=None, K=None):
    """the (preset, kind) projection, kept until another preset is asked for (bounded memory: 70B's gate/up is 0.9 GB of bf16)"""
    key = (preset, kind)
    if key not in _CACHE:
        if any(k[0] != preset for k in _CACHE):
            _CACHE.clear(); torch.cuda.empty_cache()
        if N is None:
            H, nh, nkv, D, F, _ = LAYOUTS[preset]
            N, K = {"o": (H, nh * D), "down": (H, F), "qkv": ((nh + 2 * nkv) * D, H), "gu": (2 * F, H)}[kind]
        _CACHE[key] = Proj(L, N, K, zlib.crc32(f"{preset}/{kind}".encode()) & 0xFFFF)
    return _CACHE[key]


# ------------------------------------------------------------------------------------------------ o / down: x += A.B^T; xn = rmsnorm(x) * gain
def rp_inputs(P, seed):
    g = gen(seed)
    x0 = torch.randn(MAXM, P.N, device=dev(), generator=g).to(BF16)
    gain = (1 + 0.3 * torch.randn(P.N, device=dev(), generator=g)).to(BF16)
    return x0, gain


def rp_run(L, P, M, path, bn, G, x0, gain, fp8=False, launches=1):
    A, sa, B, sb = P.ops(fp8)
    x = x0.clone()
    xn = torch.full_like(x0, float("nan"))
    rc = L.oa_k_sk_row_parallel(ptr(A), ptr(sa), ptr(B), ptr(sb), M, P.N, P.K, bn, G, path, ptr(x), ptr(gain), ptr(xn), EPS, launches, None)
    return rc, x, xn


def rp_reference_check(P, M, x0, gain, x, xn, fp8, what, min_equal):
    acc, tol = P.product(fp8, M)
    check_bf16(x[:M], x0[:M].double() + acc, f"x{'/fp8' if fp8 else ''}: {what}", abs_tol=tol, min_equal=min_equal)
    xk = x[:M].double()                                    # the norm of the kernel's own new residual row
    xnr = xk * torch.rsqrt((xk * xk).mean(1, keepdim=True) + EPS) * gain.double()
    check_bf16(xn[:M], xnr, f"xn{'/fp8' if fp8 else ''}: {what}", min_equal=min_equal)


def rp_configs(sms, fp8):
    """(path, block_n, n_ctas, M) of every variant the engine can run for a row-parallel projection"""
    cfg = []
    for M in MS:
        for G in (sms, 7):
            cfg += [(0, bn, G, M) for bn in ((64, 128) if fp8 else (64, 128, 256))] + [(1, 128, G, M)]
        if not fp8:
            cfg += [(S, 128, sms, M) for S in CLUSTERS]
    if not fp8:
        cfg += [(0, 128, G, M) for M in (129, 256) for G in (sms, 7)]      # two 128-row tiles (sk_max_rows = 256)
    return cfg


@pytest.mark.parametrize("kind", ["o", "down"])
@pytest.mark.parametrize("preset", PRESETS)
def test_row_parallel_matches_fp64(L, sms, preset, kind):
    P = proj(L, preset, kind)
    x0, gain = rp_inputs(P, 1)
    for fp8 in (False, True):
        for path, bn, G, M in rp_configs(sms, fp8):
            what = f"{preset} {kind} path {path} bn {bn} n_ctas {G} M {M}"
            rc, x, xn = rp_run(L, P, M, path, bn, G, x0, gain, fp8)
            assert rc == 0, (what, rc, _lib.last_error())
            rp_reference_check(P, M, x0, gain, x, xn, fp8, what, MIN_EQUAL_FP8 if fp8 else P.min_equal)
    report(f"{preset} {kind}")


# ------------------------------------------------------------------------------------------------ gate/up: act = silu(gate) * up
def gu_run(L, P, M, path, bn, G, fp8=False, launches=1):
    A, sa, B, sb = P.ops(fp8)
    act = torch.full((MAXM, P.N // 2), float("nan"), dtype=BF16, device=dev())
    rc = L.oa_k_sk_swiglu(ptr(A), ptr(sa), ptr(B), ptr(sb), M, P.N // 2, P.K, bn, G, path, ptr(act), launches, None)
    return rc, act


def gu_reference(P, M, fp8):
    acc, tol = P.product(fp8, M)
    r = acc.view(M, P.N // 32, 2, 16)                      # physical columns: 16 gate, then 16 up per 32
    gte, up = r[:, :, 0], r[:, :, 1]
    return (gte / (1 + torch.exp(-gte)) * up).reshape(M, P.N // 2), tol


# + a small gate/up (N = 1024, K = 4096: 512 k-block units on 132 SMs) whose tiles are cut into up to 17 pieces.  At the presets' shapes
# every CTA owns more units than a tile has, so no tile has more than two pieces there and the finisher's loop over further pieces never runs.
@pytest.mark.parametrize("preset", list(LAYOUTS) + ["many-pieces"])
def test_swiglu_matches_fp64(L, sms, preset):
    P = proj(L, preset, "gu", *((1024, 4096) if preset == "many-pieces" else (None, None)))
    for fp8 in (False, True):
        for M in MS + ([] if fp8 else [129, 256]):
            for G in (sms, 7):
                runs = [(0, bn) for bn in ((64, 128) if fp8 else (64, 128, 256))] if M <= 128 else [(0, 128)]
                if M <= 128 and not fp8:
                    runs.append((1, 128))
                ref, tol = gu_reference(P, M, fp8)
                acts = {}
                for path, bn in runs:
                    what = f"act{'/fp8' if fp8 else ''}: {preset} path {path} bn {bn} n_ctas {G} M {M}"
                    rc, act = gu_run(L, P, M, path, bn, G, fp8)
                    assert rc == 0, (what, rc, _lib.last_error())
                    acts[path, bn] = act
                    # the gate/up tolerance: silu(g) * u scales the product's error by at most max|u| ~ 5 of its rms
                    check_bf16(act[:M], ref, what, abs_tol=5 * tol, min_equal=MIN_EQUAL_FP8 if fp8 else MIN_EQUAL)
                if (1, 128) in acts:
                    assert same(acts[0, 128], acts[1, 128]), f"fused SwiGLU vs the consumer: {preset} n_ctas {G} M {M}"
    report(preset)


# ------------------------------------------------------------------------------------------------ qkv: (+ bias) -> bf16 -> RoPE -> q_out / paged KV
def rope_tables(D, theta=500000.0):
    half = D // 2
    inv = theta ** (-2.0 * torch.arange(half, dtype=torch.float64) / D)
    a = torch.arange(MAX_POS, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.cos(a).float().to(dev()).contiguous(), torch.sin(a).float().to(dev()).contiguous()


KV_SCALES = [None, (1.0, 1.0), (0.37, 2.9)]       # None: bf16 cache


class QkvCase:
    """positions / slots / RoPE tables / bias of one preset's qkv projection and a 3-layer cache whose middle layer is written (the
    outer layers stand for other layers' pages)"""
    NUM_PAGES = 12

    def __init__(self, preset, nh, nkv, D, bias, seed=7):
        self.nh, self.nkv, self.D = nh, nkv, D
        g = torch.Generator(device="cpu").manual_seed(seed)
        pos = torch.randint(0, MAX_POS, (MAXM,), generator=g, dtype=torch.int32)
        pos[::3] = 8192 + torch.randint(0, MAX_POS - 8192, (len(pos[::3]),), generator=g, dtype=torch.int32)
        self.pos = pos.to(dev())
        self.slots = torch.randperm(self.NUM_PAGES * 64, generator=g)[:MAXM].to(torch.int32).to(dev())
        self.cos, self.sin = rope_tables(D)
        N = (nh + 2 * nkv) * D
        self.bias = (torch.randn(N, generator=g) * 0.5).to(BF16).to(dev()) if bias else None

    def layer_elems(self, fp8):
        return 2 * self.NUM_PAGES * self.nkv * 64 * self.D

    def new_cache(self, fp8):
        n = self.layer_elems(fp8)
        if fp8:
            return torch.full((3 * n,), 0x7F, dtype=torch.uint8, device=dev())
        return torch.full((3 * n,), KV_FILL_BF16, dtype=torch.int16, device=dev()).view(BF16)

    def layer(self, cache, fp8):
        n = self.layer_elems(fp8)
        return cache[n:2 * n]

    def kv_rows(self, cache, fp8, M):
        """the kernel's K and V rows of the first M tokens: [M, nkv, D] (bf16 values or e4m3 bytes)"""
        lay = self.layer(cache, fp8).view(2, self.NUM_PAGES, self.nkv, -1)
        page, off = self.slots[:M].long() // 64, self.slots[:M].long() % 64
        k = lay[0].view(self.NUM_PAGES, self.nkv, 64, self.D)[page, :, off]
        v = lay[1].view(self.NUM_PAGES, self.nkv, self.D, 64)[page, :, :, off] if fp8 else lay[1].view(self.NUM_PAGES, self.nkv, 64, self.D)[page, :, off]
        return k, v

    def untouched(self, cache, fp8, M, what):
        """every cache element outside the rows of slots[:M] of the middle layer still holds the sentinel"""
        fill = 0x7F if fp8 else KV_FILL_BF16
        raw = cache if fp8 else cache.view(torch.int16)
        n = self.layer_elems(fp8)
        assert (raw[:n] == fill).all() and (raw[2 * n:] == fill).all(), f"{what}: another layer's pages changed"
        lay = raw[n:2 * n].view(2, self.NUM_PAGES, self.nkv, -1)
        written = torch.zeros(self.NUM_PAGES, 64, dtype=torch.bool, device=dev())
        written[self.slots[:M].long() // 64, self.slots[:M].long() % 64] = True
        k = lay[0].view(self.NUM_PAGES, self.nkv, 64, self.D).permute(0, 2, 1, 3)
        v = (lay[1].view(self.NUM_PAGES, self.nkv, self.D, 64).permute(0, 3, 1, 2) if fp8 else
             lay[1].view(self.NUM_PAGES, self.nkv, 64, self.D).permute(0, 2, 1, 3))
        assert (k[~written] == fill).all() and (v[~written] == fill).all(), f"{what}: a KV row outside `slots` changed"
        assert (k[written] != fill).all() and (v[written] != fill).all(), f"{what}: a KV row in `slots` was not written"

    def reference(self, s64, delta, M):
        """fp64 reference of the qkv finish from the projection + bias s64 [M, N]: the kernel rounds its fp32 sum to bf16 before RoPE, and
        that sum may land on either side of a bf16 rounding boundary within `delta` of the fp64 value, so each pre-RoPE value is the
        interval [bf16(s - delta), bf16(s + delta)] and each rotated value the interval of the rotation over those.  Returns
        (center, lo, hi) as [M, nh + 2 nkv, D], center = the rotation of bf16(s)."""
        D, half = self.D, self.D // 2
        heads = self.nh + 2 * self.nkv
        v = s64.to(BF16).double().view(M, heads, D)
        va = (s64 - delta).to(BF16).double().view(M, heads, D)
        vb = (s64 + delta).to(BF16).double().view(M, heads, D)
        c = self.cos[self.pos[:M].long()].double()[:, None, :]
        s = self.sin[self.pos[:M].long()].double()[:, None, :]
        nr = self.nh + self.nkv

        def rot(t):
            lo, hi = t[:, :nr, :half], t[:, :nr, half:]
            return lo * c - hi * s, hi * c + lo * s

        def span(a, b):
            return torch.minimum(a, b), torch.maximum(a, b)

        ca, cb = rot(v)
        lo_a, lo_b = span(va[:, :nr, :half] * c, vb[:, :nr, :half] * c)
        hi_a, hi_b = span(va[:, :nr, half:] * s, vb[:, :nr, half:] * s)
        hc_a, hc_b = span(va[:, :nr, half:] * c, vb[:, :nr, half:] * c)
        ls_a, ls_b = span(va[:, :nr, :half] * s, vb[:, :nr, :half] * s)
        center = torch.cat([torch.cat([ca, cb], -1), v[:, nr:]], 1)
        lo = torch.cat([torch.cat([lo_a - hi_b, hc_a + ls_a], -1), va[:, nr:]], 1)
        hi = torch.cat([torch.cat([lo_b - hi_a, hc_b + ls_b], -1), vb[:, nr:]], 1)
        return center, lo, hi


def q8(x, scale):
    """the byte an fp8 writer stores for x (fp32 math): e4m3(x * (1/scale)), saturating"""
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(scale, dtype=torch.float32)
    return (x.float() * inv.to(x.device)).clamp(-448, 448).to(FP8)


def qkv_run(L, P, Q, M, path, bn, G, kvs, fp8=False):
    A, sa, B, sb = P.ops(fp8)
    q_out = torch.full((MAXM, Q.nh * Q.D), float("nan"), dtype=BF16, device=dev())
    cache = Q.new_cache(kvs is not None)
    ks, vs = kvs if kvs else (0.0, 0.0)
    rc = L.oa_k_sk_qkv_rope(ptr(A), ptr(sa), ptr(B), ptr(sb), ptr(Q.bias), M, P.K, Q.nh, Q.nkv, Q.D, bn, G, path, ptr(Q.pos), ptr(Q.slots),
                            ptr(Q.cos), ptr(Q.sin), ptr(q_out), ptr(Q.layer(cache, kvs is not None)), Q.NUM_PAGES, ks, vs, None)
    return rc, q_out, cache


def qkv_check(P, Q, M, q_out, cache, kvs, fp8, what, min_equal):
    acc, tol = P.product(fp8, M)
    s64 = acc + (Q.bias.double() if Q.bias is not None else 0.0)
    center, lo, hi = Q.reference(s64, tol, M)
    nh, nkv = Q.nh, Q.nkv
    tag = "/fp8" if fp8 else ""
    check_bf16(q_out[:M].view(M, nh, Q.D), center[:, :nh], f"q{tag}: {what}", lo[:, :nh], hi[:, :nh], abs_tol=tol, min_equal=min_equal)
    kk, vv = Q.kv_rows(cache, kvs is not None, M)
    if kvs is None:
        check_bf16(kk, center[:, nh:nh + nkv], f"k{tag}: {what}", lo[:, nh:nh + nkv], hi[:, nh:nh + nkv], abs_tol=tol, min_equal=min_equal)
        check_bf16(vv, center[:, nh + nkv:], f"v{tag}: {what}", lo[:, nh + nkv:], hi[:, nh + nkv:], min_equal=min_equal)
    else:
        # fp8 cache: the kernel's bf16 value is one the bounds above allow, and e4m3(value / s) is monotone in it, so each byte lies between
        # the bytes of the interval's ends (the three-neighbour rule of test_fp8_kv_write over the interval)
        for name, got, sl, sc, extra in (("k8", kk, slice(nh, nh + nkv), kvs[0], 1), ("v8", vv, slice(nh + nkv, None), kvs[1], 0)):
            c, a, b = center[:, sl], lo[:, sl], hi[:, sl]
            u = torch.maximum(ulp(torch.maximum(a.abs(), b.abs())), torch.full_like(a, tol)) * extra
            g8 = got.view(FP8).double()
            lo8, hi8 = q8((a - u).to(BF16), sc).double(), q8((b + u).to(BF16), sc).double()
            bad = ~((g8 >= lo8) & (g8 <= hi8))
            assert not bad.any(), f"{name}{tag}: {what}: {int(bad.sum())} bytes outside their reference interval"
            frac = (got.view(torch.uint8) == q8(c.to(BF16), sc).view(torch.uint8)).double().mean().item()
            MATCH[name + tag] = min(MATCH.get(name + tag, 1.0), frac)
            assert frac >= min_equal, f"{name}{tag}: {what}: only {frac:.5f} of the bytes equal the rounded reference's"


@pytest.mark.parametrize("preset", LAYOUTS)
def test_qkv_rope_kv_write_matches_fp64(L, sms, preset):
    H, nh, nkv, D, F, bias = LAYOUTS[preset]
    P = proj(L, preset, "qkv")
    Q = QkvCase(preset, nh, nkv, D, bias)
    for fp8 in (False, True):
        for kvs in KV_SCALES:
            cfg = []
            for M in MS:
                for G in (sms, 7):
                    cfg += [(0, bn, G, M) for bn in ((64, 128) if fp8 else (64, 128, 256))] + [(1, 128, G, M)]
                if not fp8:
                    cfg += [(S, 128, sms, M) for S in CLUSTERS]
            if not fp8:
                cfg += [(0, 128, G, M) for M in (129, 256) for G in (sms, 7)]
            for path, bn, G, M in cfg:
                what = f"{preset} cache {kvs or 'bf16'} path {path} bn {bn} n_ctas {G} M {M}"
                rc, q_out, cache = qkv_run(L, P, Q, M, path, bn, G, kvs, fp8)
                assert rc == 0, (what, rc, _lib.last_error())
                # the K / V rows of one or two tokens of a tensor-parallel rank (one or two kv heads) are 128 to 256 values: too few for
                # an exact-match floor (two misses fail 0.99).  Every preset's rows have at least 512.
                floor = (MIN_EQUAL_FP8 if fp8 else MIN_EQUAL) if M * nkv * D >= 512 else 0.0
                qkv_check(P, Q, M, q_out, cache, kvs, fp8, what, floor)
    report(preset)


# ------------------------------------------------------------------------------------------------ stream-K: fused == stand-alone, bit for bit
@pytest.mark.parametrize("preset", PRESETS)
def test_stream_k_fused_finishers_equal_the_consumers(L, sms, preset):
    """paths 0 and 1 at block_n 128 add the same partials in the same CTA order and finish with the same helpers: bit-identical results.
    Both also equal the bf16 rounding of the stand-alone fixed-order partial sum (oa_k_gemm_streamk) where the finish is one exact add."""
    H, nh, nkv, D, F, bias = PRESETS[preset]
    Po, Pg, Pq = proj(L, preset, "o"), proj(L, preset, "gu"), proj(L, preset, "qkv")
    Q = QkvCase(preset, nh, nkv, D, bias)
    x0, gain = rp_inputs(Po, 2)
    for M in MS:
        for G in (sms, 7):
            what = f"{preset} n_ctas {G} M {M}"
            for fp8 in (False, True):
                runs = [rp_run(L, Po, M, p, 128, G, x0, gain, fp8) for p in (0, 1)]
                assert runs[0][0] == 0 and runs[1][0] == 0, what
                assert same(runs[0][1], runs[1][1]) and same(runs[0][2], runs[1][2]), f"o finish, fp8 {fp8}: {what}"
                A, sa, B, sb = Po.ops(fp8)
                s32 = torch.empty(M, Po.N, dtype=torch.float32, device=dev())
                rc = (L.oa_k_gemm_streamk_fp8(ptr(A), ptr(sa), ptr(B), ptr(sb), M, Po.N, Po.K, 128, G, 0, None, ptr(s32), None) if fp8 else
                      L.oa_k_gemm_streamk(ptr(A), ptr(B), M, Po.N, Po.K, 128, G, ptr(s32), None))
                assert rc == 0
                assert torch.equal(runs[0][1][:M], (s32 + x0[:M].float()).to(BF16)), f"o finish vs the partial sum, fp8 {fp8}: {what}"
                for kvs in KV_SCALES:
                    r0, r1 = (qkv_run(L, Pq, Q, M, p, 128, G, kvs, fp8) for p in (0, 1))
                    assert r0[0] == 0 and r1[0] == 0, what
                    assert same(r0[1], r1[1]) and same(r0[2], r1[2]), \
                        f"qkv finish, fp8 {fp8}, cache {kvs}: {what}"
            a0, a1 = gu_run(L, Pg, M, 0, 128, G), gu_run(L, Pg, M, 1, 128, G)
            assert a0[0] == 0 and a1[0] == 0, what
            assert same(a0[1], a1[1]), f"gate/up finish: {what}"


# ------------------------------------------------------------------------------------------------ cluster split-K vs stream-K
CK_SHAPES = [("llama-3.2-1b", None), ("llama-3-8b", None), ("custom-d64-odd", (1024, 5, 1, 64))]     # custom: N = 7 * 64, not a multiple of 128


@pytest.mark.parametrize("preset,shape", CK_SHAPES)
def test_cluster_k_within_one_ulp_of_stream_k(L, sms, preset, shape):
    if shape is None:
        H, nh, nkv, D, F, bias = PRESETS[preset]
    else:
        (H, nh, nkv, D), bias = shape, False
    N = (nh + 2 * nkv) * D
    Pq = proj(L, preset, "qkv", N, H)
    Po = proj(L, preset, "o", H, H if shape else nh * D)       # K >= 8 k blocks for S = 8
    Q = QkvCase(preset, nh, nkv, D, bias)
    x0, gain = rp_inputs(Po, 3)
    for M in (1, 64, 127, 128):
        _, xs, _ = rp_run(L, Po, M, 0, 128, sms, x0, gain)
        _, qs, cs = qkv_run(L, Pq, Q, M, 0, 128, sms, None)
        ks, vs = Q.kv_rows(cs, False, M)
        acc, tol = Pq.product(False, M)
        center, lo, hi = Q.reference(acc + (Q.bias.double() if Q.bias is not None else 0.0), tol, M)
        width = hi - lo                                       # the pre-RoPE rounding may differ between two fp32 sums
        for S in CLUSTERS:
            what = f"{preset} S {S} M {M}"
            rc, xc, _ = rp_run(L, Po, M, S, 128, sms, x0, gain)
            assert rc == 0, (what, _lib.last_error())
            check_bf16(xc[:M], xs[:M].double(), f"x cluster-K vs stream-K: {what}", abs_tol=Po.tol, min_equal=MIN_EQUAL)
            # (xn is the norm of a different x: test_row_parallel_matches_fp64 checks it against the fp64 norm of the cluster path's own x)
            rc, qc, cc = qkv_run(L, Pq, Q, M, S, 128, sms, None)
            assert rc == 0, (what, _lib.last_error())
            kc, vc = Q.kv_rows(cc, False, M)
            nr = nh + nkv
            for name, a, b, w in (("q", qc[:M].view(M, nh, D), qs[:M].view(M, nh, D), width[:, :nh]), ("k", kc, ks, width[:, nh:nr]),
                                  ("v", vc, vs, width[:, nr:])):
                ref = b.double()
                check_bf16(a, ref, f"{name} cluster-K vs stream-K: {what}", ref - w, ref + w, abs_tol=Pq.tol, min_equal=MIN_EQUAL)
            Q.untouched(cc, False, M, what)
    report(preset)


# ------------------------------------------------------------------------------------------------ reproducibility and the flags' re-arm
@pytest.mark.parametrize("preset", ["llama-3.2-1b", "llama-3-70b"])
def test_repeated_launches_are_bitwise_reproducible(L, sms, preset):
    """a second call gives the same bits, and `launches = 2` on one set of tile flags (the engine's per-layer reuse) equals two calls"""
    H, nh, nkv, D, F, bias = PRESETS[preset]
    Po, Pg, Pq = proj(L, preset, "o"), proj(L, preset, "gu"), proj(L, preset, "qkv")
    Q = QkvCase(preset, nh, nkv, D, bias)
    x0, gain = rp_inputs(Po, 4)
    for M in (5, 128):
        for G in (sms, 7):
            for path in (0, 1, 4):
                what = f"{preset} path {path} n_ctas {G} M {M}"
                _, x1, xn1 = rp_run(L, Po, M, path, 128, G, x0, gain)
                _, x1b, xn1b = rp_run(L, Po, M, path, 128, G, x0, gain)
                assert same(x1, x1b) and same(xn1, xn1b), f"second call: {what}"
                rc, x2, xn2 = rp_run(L, Po, M, path, 128, G, x0, gain, launches=2)
                assert rc == 0
                _, x2b, xn2b = rp_run(L, Po, M, path, 128, G, x1, gain)
                assert same(x2, x2b) and same(xn2, xn2b), f"launches = 2 vs two calls: {what}"
                acc, tol = Po.product(False, M)                # ... and the reference applied twice
                check_bf16(x2[:M], x1[:M].double() + acc, f"x twice: {what}", abs_tol=tol)
                r1, r2 = qkv_run(L, Pq, Q, M, path, 128, G, (0.37, 2.9) if path != 4 else None), \
                    qkv_run(L, Pq, Q, M, path, 128, G, (0.37, 2.9) if path != 4 else None)
                assert same(r1[1], r2[1]) and same(r1[2], r2[2]), f"qkv: {what}"
            for path in (0, 1):
                _, a1 = gu_run(L, Pg, M, path, 128, G)
                rc, a2 = gu_run(L, Pg, M, path, 128, G, launches=2)
                assert rc == 0 and same(a1, a2), f"gate/up launches = 2: {preset} path {path} n_ctas {G} M {M}"


# ------------------------------------------------------------------------------------------------ nothing outside the written region
@pytest.mark.parametrize("preset", ["llama-3.2-1b", "qwen2.5-32b", "llama-3-70b"])
def test_writes_stay_inside_their_rows(L, sms, preset):
    H, nh, nkv, D, F, bias = PRESETS[preset]
    Po, Pg, Pq = proj(L, preset, "down"), proj(L, preset, "gu"), proj(L, preset, "qkv")
    Q = QkvCase(preset, nh, nkv, D, bias)
    x0, gain = rp_inputs(Po, 5)
    nan = torch.tensor(BF16_NAN, dtype=torch.int16, device=dev())
    for M in (1, 5, 127, 129):
        for path in ((0,) if M > 128 else (0, 1, 2, 8)):
            what = f"{preset} path {path} M {M}"
            rc, x, xn = rp_run(L, Po, M, path, 128, sms, x0, gain)
            assert rc == 0, what
            assert torch.equal(x[M:], x0[M:]) and (xn[M:].view(torch.int16) == nan).all(), f"x / xn rows >= M: {what}"
            assert not (xn[:M].view(torch.int16) == nan).any(), f"xn rows < M: {what}"
            if path <= 1:
                rc, act = gu_run(L, Pg, M, path, 128, sms)
                assert rc == 0 and (act[M:].view(torch.int16) == nan).all() and not (act[:M].view(torch.int16) == nan).any(), f"act: {what}"
            for kvs in ((None, (0.37, 2.9)) if path <= 1 else (None,)):
                rc, q_out, cache = qkv_run(L, Pq, Q, M, path, 128, sms, kvs)
                assert rc == 0, what
                assert (q_out[M:].view(torch.int16) == nan).all() and not (q_out[:M].view(torch.int16) == nan).any(), f"q_out: {what}"
                Q.untouched(cache, kvs is not None, M, f"{what} cache {kvs}")


# ------------------------------------------------------------------------------------------------ refusals
def test_launchers_refuse_what_they_cannot_run(L, sms):
    """every refusal happens on the host, before a launch: nothing below reaches a kernel, and no output changes"""
    P = proj(L, "llama-3.2-1b", "o")
    Pg = proj(L, "llama-3.2-1b", "gu")
    Pq = proj(L, "llama-3.2-1b", "qkv")
    Q = QkvCase("llama-3.2-1b", 32, 8, 64, False)
    x0, gain = rp_inputs(P, 6)
    BAD = _lib.OA_ERR_BAD_REQUEST

    def rp(M, path, G=sms, fp8=False, K=None):
        A, sa, B, sb = P.ops(fp8)
        x = x0.clone(); xn = torch.zeros_like(x0)
        rc = L.oa_k_sk_row_parallel(ptr(A), ptr(sa), ptr(B), ptr(sb), M, P.N, K or P.K, 128, G, path, ptr(x), ptr(gain), ptr(xn), EPS, 1, None)
        assert torch.equal(x, x0) and not xn.any(), (M, path, G, fp8, K)
        return rc

    def qk(M, path, G=sms, fp8=False, K=None):
        A, sa, B, sb = Pq.ops(fp8)
        q_out = torch.zeros(MAXM, Q.nh * Q.D, dtype=BF16, device=dev())
        cache = Q.new_cache(False)
        rc = L.oa_k_sk_qkv_rope(ptr(A), ptr(sa), ptr(B), ptr(sb), None, M, K or Pq.K, Q.nh, Q.nkv, Q.D, 128, G, path, ptr(Q.pos), ptr(Q.slots),
                                ptr(Q.cos), ptr(Q.sin), ptr(q_out), ptr(Q.layer(cache, False)), Q.NUM_PAGES, 0.0, 0.0, None)
        assert not q_out.any() and (cache.view(torch.int16) == KV_FILL_BF16).all()
        return rc

    def gu(M, path, G=sms, fp8=False):
        A, sa, B, sb = Pg.ops(fp8)
        act = torch.zeros(MAXM, Pg.N // 2, dtype=BF16, device=dev())
        rc = L.oa_k_sk_swiglu(ptr(A), ptr(sa), ptr(B), ptr(sb), M, Pg.N // 2, Pg.K, 128, G, path, ptr(act), 1, None)
        assert not act.any()
        return rc

    # the fused finishers: one 128-row tile, every CTA resident (finishing CTAs wait for the others), no fp8 SwiGLU finisher
    assert rp(129, 1) == BAD and qk(129, 1) == BAD and gu(129, 1) == BAD
    assert rp(128, 1, G=sms + 1) == BAD and qk(128, 1, G=sms + 1) == BAD and gu(128, 1, G=sms + 1) == BAD
    assert gu(5, 1, fp8=True) == BAD
    # cluster split-K: S in {2, 3, 4, 8}, one row tile, bf16, and at least one 64-wide k block per CTA of a cluster
    for S in (5, 6, 7, 16):
        assert rp(5, S) == BAD and qk(5, S) == BAD
    assert rp(129, 4) == BAD and qk(129, 4) == BAD and rp(5, 4, fp8=True) == BAD and qk(5, 4, fp8=True) == BAD
    for K, S in ((64, 2), (128, 3), (192, 4), (448, 8)):
        assert rp(5, S, K=K) == BAD and qk(5, S, K=K) == BAD, (K, S)


# ------------------------------------------------------------------------------------------------ decode attention with the in-kernel merge
CTX = [1, 63, 64, 65, 1000, 1790, 129, 517, 1600, 1701, 2, 333, 9000]


def attn_ref64(q, K, V, bt, ctx, nh, nkv, D):
    """fp64 softmax attention of one query row per sequence over its first ctx tokens.  K, V: [pages, nkv, 64, D] as the kernel reads them"""
    grp = nh // nkv
    outs = []
    for i, c in enumerate(ctx):
        pages = bt[i, : (c + 63) // 64]
        k = K[pages].permute(0, 2, 1, 3).reshape(-1, nkv, D)[:c].double().repeat_interleave(grp, 1)
        v = V[pages].permute(0, 2, 1, 3).reshape(-1, nkv, D)[:c].double().repeat_interleave(grp, 1)
        s = torch.einsum("hd,khd->hk", q[i].double(), k) / D ** 0.5
        outs.append(torch.einsum("hk,khd->hd", torch.softmax(s, -1), v))
    return torch.stack(outs)


@pytest.mark.parametrize("kvs", KV_SCALES)
@pytest.mark.parametrize("nh,nkv,D", [(8, 8, 128), (32, 8, 64), (32, 8, 128), (40, 8, 128), (64, 8, 128),    # GQA groups 1, 4, 4, 5, 8
                                      (10, 2, 128), (8, 1, 128)])       # one tensor-parallel rank of Qwen2.5-32B t = 4, Llama-3-70B t = 8
def test_decode_attention_in_kernel_merge(L, sms, nh, nkv, D, kvs):
    n = len(CTX); maxp = max((c + 63) // 64 for c in CTX); num_pages = sum((c + 63) // 64 for c in CTX) + 7
    g = torch.Generator(device="cpu").manual_seed(nh + D)
    kv = torch.randn(2, num_pages, nkv, 64, D, generator=g).to(BF16).to(dev())
    if kvs:
        ks, vs = kvs
        k8, v8 = q8(kv[0] * ks * 2, ks), q8(kv[1] * ks * 2, vs)          # the magnitudes of test_fp8_paged_decode_attention
        cache = torch.stack([k8.view(torch.uint8).reshape(num_pages, nkv, 64 * D),
                             v8.view(torch.uint8).transpose(2, 3).contiguous().reshape(num_pages, nkv, 64 * D)]).contiguous()
        Kd, Vd = k8.float().double() * ks, v8.float().double() * vs
    else:
        ks, vs = 0.0, 0.0
        cache, Kd, Vd = kv, kv[0], kv[1]
    perm = torch.randperm(num_pages, generator=g)
    bt = torch.zeros(n, maxp, dtype=torch.int32); k = 0
    for i, c in enumerate(CTX):
        npg = (c + 63) // 64; bt[i, :npg] = perm[k:k + npg].to(torch.int32); k += npg
    q = torch.randn(n, nh, D, generator=g).to(BF16).to(dev())
    ctx_a = np.array(CTX, np.int32); bt_np = np.ascontiguousarray(bt.numpy())

    def run(target, inline, launches):
        out = torch.full((n, nh, D), float("nan"), dtype=BF16, device=dev())
        rc = L.oa_k_decode_attention(ptr(q), ptr(out), ptr(cache), num_pages, bt_np.ctypes.data, maxp, ctx_a.ctypes.data, n, nh, nkv, D,
                                     target, inline, launches, ks, vs, None)
        assert rc == 0, _lib.last_error()
        return out

    out1 = run(2 * sms, 1, 1)
    ref = attn_ref64(q, Kd, Vd, bt.to(dev()).long(), CTX, nh, nkv, D)
    vscale = vs if kvs else 1.0
    assert torch.isfinite(out1.float()).all()
    err = ((out1.double() - ref) / vscale).abs().max().item()          # in units of the V scale
    assert err < 2e-2, err
    # the counters advance by n_pieces per launch: three launches on one counter array merge every cut item each time
    assert torch.equal(run(2 * sms, 1, 3), out1)
    # the separate merge kernel on the same plan divides by l where the in-kernel merge multiplies by 1/l: 1 ulp apart at most
    for target in (2 * sms, 2 * 132, 7):
        a, b = run(target, 1, 1), run(target, 0, 1)
        d = (a.double() - b.double()).abs()
        assert (d <= ulp(torch.maximum(a.double().abs(), b.double().abs()))).all(), (target, d.max().item())
        assert ((a.double() - ref) / vscale).abs().max().item() < 2e-2, target
    # ... which is what oa_k_paged_attention runs (a plan for 2 x 132 CTAs)
    sep = torch.full((n, nh, D), float("nan"), dtype=BF16, device=dev())
    ql = np.ones(n, np.int32)
    args = (ptr(q), ptr(sep), ptr(cache), num_pages, bt_np.ctypes.data, maxp, ctx_a.ctypes.data, ql.ctypes.data, n, nh, nkv, D, 0)
    assert (L.oa_k_paged_attention_fp8(*args, ks, vs, None) if kvs else L.oa_k_paged_attention(*args, None)) == 0
    a = run(2 * 132, 1, 1)
    assert (((a.double() - sep.double()).abs()) <= ulp(torch.maximum(a.double().abs(), sep.double().abs()))).all()


# ------------------------------------------------------------------------------------------------ LM head: grammar-masked arg-max
@pytest.mark.parametrize("V,shard,col_offset", [(128256, 1, 0), (152064, 1, 0), (128256, 8, 3 * 128256 // 8), (152064, 8, 7 * 152064 // 8),
                                                (128256, 8, 8), (152064, 8, 24)])
def test_masked_argmax(L, V, shard, col_offset):
    """a vocabulary shard of N = V / shard columns whose first global id is col_offset (offsets 8 and 24 are not word-aligned)"""
    N, K, M = V // shard, 512, 12
    words = (V + 31) // 32
    g = torch.Generator(device="cpu").manual_seed(V + col_offset)
    A = torch.randn(M, K, generator=g).to(BF16)
    B = (torch.randn(N, K, generator=g) * 0.1).to(BF16)
    j1, j2, j3 = 3 * N // 10, N - 300, N // 2 + 5
    B[j2] = B[j1]; B[j3 + 1] = B[j3]                  # exact ties: across tiles, and inside one 32-column chunk
    A, B = A.to(dev()), B.to(dev())
    bits = np.zeros((6, words * 32), np.bool_)
    rng = np.random.default_rng(V)
    bits[0] = rng.random(words * 32) < 0.3            # a sparse grammar state
    bits[1, col_offset + N - 1] = True                 # a single id: the shard's last column (the last, partial, tile)
    w = ((col_offset + N // 3) // 32 + 1) * 32         # ids straddling a 32-id word of the bitset
    bits[2, w - 3:w + 2] = True
    bits[2, col_offset + 40] = True
    # slot 3 allows nothing
    bits[4, [col_offset + j1, col_offset + j2]] = True
    bits[5, [col_offset + j3, col_offset + j3 + 1]] = True
    bits[:, V:] = False
    table = torch.from_numpy(np.packbits(bits, axis=1, bitorder="little").view(np.int32).copy()).to(dev())
    slot = torch.tensor([-1, 0, 1, 2, 3, 4, 5, -1, 0, 2, 1, 4], dtype=torch.int32, device=dev())
    ref = A.double() @ B.double().T
    allowed = torch.from_numpy(bits[:, col_offset:col_offset + N].copy()).to(dev())
    for bn in (64, 128, 256):
        logits = torch.full((M, N), float("nan"), dtype=torch.float32, device=dev())
        ids = torch.full((M,), -1, dtype=torch.int32, device=dev())
        rc = L.oa_k_gemm_logits_masked(ptr(A), ptr(B), M, N, K, bn, ptr(table), ptr(slot), words, col_offset, ptr(logits), ptr(ids), None)
        assert rc == 0, _lib.last_error()
        assert ((logits.double() - ref).abs() <= 1e-4 * K ** 0.5 + 1e-5 * ref.abs()).all()
        assert torch.equal(logits[:, j1], logits[:, j2]) and torch.equal(logits[:, j3], logits[:, j3 + 1])
        ok = torch.ones(M, N, dtype=torch.bool, device=dev())
        masked = slot >= 0
        ok[masked] = allowed[slot[masked].long()]
        lg = torch.where(ok, logits, torch.tensor(-float("inf"), device=dev()))
        mx = lg.max(1, keepdim=True).values
        first = torch.where(ok & (lg == mx), torch.arange(N, device=dev())[None, :], N).min(1).values
        exp = torch.where(first == N, 0, first)        # a row allowing nothing takes id 0
        assert torch.equal(ids.long(), exp), (bn, ids.tolist(), exp.tolist())
        assert ids[2].item() == N - 1 and ids[4].item() == 0 and ids[5].item() == j1 and ids[11].item() == j1 and ids[6].item() == j3


# ------------------------------------------------------------------------------------------------ the prefill KV writer on a bf16 cache
@pytest.mark.parametrize("nh,nkv,D", [(32, 8, 64), (32, 8, 128), (40, 8, 128), (5, 1, 64)])
def test_kv_write_bf16(L, nh, nkv, D):
    T = 150
    g = torch.Generator(device="cpu").manual_seed(nh * D)
    qkv = (torch.randn(T, (nh + 2 * nkv) * D, generator=g) * 3).to(BF16).to(dev())
    Q = QkvCase("kv", nh, nkv, D, False, seed=nh + D)
    pos, slots = Q.pos[:T], Q.slots[:T]
    q_out = torch.full((T + 4, nh * D), float("nan"), dtype=BF16, device=dev())
    cache = Q.new_cache(False)
    assert L.oa_k_kv_write(ptr(qkv), ptr(pos), ptr(slots), ptr(Q.cos), ptr(Q.sin), ptr(q_out), ptr(Q.layer(cache, False)), Q.NUM_PAGES, T,
                           nh, nkv, D, None) == 0
    center, lo, hi = Q.reference(qkv.double(), 0.0, T)        # qkv is bf16 already: no pre-RoPE rounding
    tol = 2.0 ** -20 * qkv.float().abs().max().item()         # the fp32 rotation's error where lo * c - hi * s cancels
    check_bf16(q_out[:T].view(T, nh, D), center[:, :nh], f"q: kv write {nh}/{nkv}/{D}", abs_tol=tol)
    k, v = Q.kv_rows(cache, False, T)
    check_bf16(k, center[:, nh:nh + nkv], f"k: kv write {nh}/{nkv}/{D}", abs_tol=tol)
    assert torch.equal(v, qkv.view(T, nh + 2 * nkv, D)[:, nh + nkv:]), "V is copied bit for bit"
    assert (q_out[T:].view(torch.int16) == BF16_NAN).all()
    Q.untouched(cache, False, T, "kv write")
    report(f"kv write {nh}/{nkv}/{D}")
