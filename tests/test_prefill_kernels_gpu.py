"""The prefill and mixed step's kernels at the single-GPU presets' shapes (pytest -m gpu): the tile and persistent projection GEMMs (store + bias,
in-place residual, SwiGLU) above 128 rows at the production K, prefill attention (and decode attention next to it in a mixed step) over
contexts up to 16384 tokens, the prefill KV writer on a pool of more than 2 GiB, RMSNorm, the embedding gather and the masked LM head.  Each
runs through the C entry point that launches it as DeviceModel::forward does.

Every family is checked twice: on operands where every intermediate is exact, so that any indexing error changes bits (compared bit for bit,
or within 1 ulp of fp64 where the kernel evaluates a transcendental), and on random operands against an fp64 reference with bounds that
scale with the reference.

The bounds come from kernel_ref.py.  Measured on an H100 80GB HBM3 (SXM, 132 SMs) at a 400 W power limit, where the file runs in about
55 s.  Smallest exact-match fractions of the random-operand projections (over every M, BLOCK_N and kernel): bf16 0.9917 at K <= 16384
(gate/up of Llama-3-70B, down of Llama-3-8B), 0.9851 and 0.9856 for the down projections of Llama-3-70B and Qwen2.5-32B (K = 28672, 27648);
e4m3 0.886 (gate/up), 0.933 (qkv), 0.947 (o, down).  RMSNorm and the KV writer's q and k: 0.99999.  Attention on random data: largest
error 1.8e-2 to 2.1e-2 of the row's rms, bf16 and fp8 caches alike (output rounding and the bf16 probabilities)."""
import ctypes as C
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from opsagent_b200 import _lib  # noqa: E402
from kernel_ref import (ACC_TOL_BF16_PER_K, ACC_TOL_FP8, BF16, FP8, MATCH, MIN_EQUAL, MIN_EQUAL_FP8, MIN_EQUAL_LONG_K,  # noqa: E402
                        check_bf16, dev, ptr, quant, report, same, ulp)

BF16_NAN = 0x7FC0            # output sentinel: rows the kernel must not write keep these bits
EPS = 1e-5
MAX_POS = 16384
A_ROWS = 8192 + 64           # the engine's activation maps span max_step_tokens rows: rows >= M hold stale data
PAD = 64                     # sentinel rows after M in every output
MS = [129, 257, 1000, 1623, 8192]
MS_FP8 = [200, 256]          # fp8 weights leave the stream-K path above 128 rows
OTHER_BN_MS = (257, 1623)    # M values that also run every BN the engine did not choose
BNS = {False: (32, 64, 128, 256), True: (32, 64, 128)}
JUNK = 3.0e4                 # large finite stale rows / pages

# name: (hidden, n_heads, n_kv, head_dim, ffn, qkv bias) of the single-GPU presets (csrc/config.hpp)
PRESETS = {
    "llama-3.2-1b": (2048, 32, 8, 64, 8192, False),
    "llama-3-8b": (4096, 32, 8, 128, 14336, False),
    "qwen2.5-32b": (5120, 40, 8, 128, 27648, True),
    "llama-3-70b": (8192, 64, 8, 128, 28672, False),
}
KINDS = {"qkv": 0, "o": 1, "gu": 2, "down": 1}       # the epilogue each projection runs on the tile path

# Attention on random data: largest |kernel - fp64| over the rms of the reference's (row, head), measured at most 2.05e-2 (see above)
ATTN_REL_TOL = 3e-2


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


def seed_of(*key):
    return zlib.crc32("/".join(map(str, key)).encode()) & 0xFFFF


def proj_shape(preset, kind):
    H, nh, nkv, D, F, _ = PRESETS[preset]
    return {"qkv": ((nh + 2 * nkv) * D, H), "o": (H, nh * D), "gu": (2 * F, H), "down": (H, F)}[kind]


def pick_bn(L, M, N, sm_count, fp8):
    return L.oa_host_pick_bn(M, N, sm_count, 0, 1 if fp8 else 0)


# ------------------------------------------------------------------------------------------------ projections
class Operands:
    """A [A_ROWS, K] (rows >= 8192 junk) and B [N, K] in bf16 and as quantised e4m3 rows, their fp64 product [8192, N] and an integer-valued
    residual / bias.  exact: sparse small-integer A (16 entries of +-1, +-2 per row, summed where they collide) and B in [-2, 2], so
    |A.B^T| <= 64, the residual and bias are integers in [-64, 64] and every sum stays below 256: exact in fp32, bf16 and the fp8 MMA."""

    def __init__(self, L, N, K, exact, seed):
        g = gen(seed)
        R = 8192
        if exact:
            A = torch.zeros(R, K, device=dev())
            cols = torch.randint(0, K, (R, 16), device=dev(), generator=g)
            vals = torch.randint(1, 3, (R, 16), device=dev(), generator=g).float() * (torch.randint(0, 2, (R, 16), device=dev(), generator=g) * 2 - 1)
            A.scatter_add_(1, cols, vals)
            B = torch.randint(-2, 3, (N, K), device=dev(), generator=g).float()
            self.resid = torch.randint(-64, 65, (R + PAD, N), device=dev(), generator=g).to(BF16)
            self.bias = torch.randint(-64, 65, (N,), device=dev(), generator=g).to(BF16)
        else:
            A = torch.randn(R, K, device=dev(), generator=g)
            B = torch.randn(N, K, device=dev(), generator=g) * K ** -0.5
            self.resid = torch.randn(R + PAD, N, device=dev(), generator=g).to(BF16)
            self.bias = (0.5 * torch.randn(N, device=dev(), generator=g)).to(BF16)
        junk = (JUNK * torch.randn(A_ROWS - R, K, device=dev(), generator=g)).to(BF16)
        self.A = torch.cat([A.to(BF16), junk])
        self.B = B.to(BF16)
        self.A8, self.sa, _ = quant(L, self.A)
        self.B8, self.sb, b8 = quant(L, self.B)
        self.junk_rows = (JUNK * torch.randn(A_ROWS, K, device=dev(), generator=g)).to(BF16)
        self.J8, self.sj, _ = quant(L, self.junk_rows)
        self.exact = exact
        self.acc = self.A[:R].double() @ self.B.double().T
        if exact:
            self.acc8 = self.acc                              # power-of-two row scales: the e4m3 copies hold the same integers
        else:
            self.acc8 = (self.A8[:R].view(FP8).double() * self.sa[:R].double()[:, None]) @ b8.T
        del b8
        self.tol = ACC_TOL_BF16_PER_K * K * self.acc.pow(2).mean().sqrt().item()
        self.tol8 = ACC_TOL_FP8 * self.acc8.abs().max().item()

    def a_operand(self, fp8, M):
        """A with rows >= M replaced by large finite junk (bf16), or its e4m3 rows and scales"""
        if fp8:
            return torch.cat([self.A8[:M], self.J8[M:]]), torch.cat([self.sa[:M], self.sj[M:]])
        return torch.cat([self.A[:M], self.junk_rows[M:]]), None


_CACHE = {}


def operands(L, preset, kind, exact):
    key = (preset, kind, exact)
    if key not in _CACHE:
        _CACHE.clear(); torch.cuda.empty_cache()
        N, K = proj_shape(preset, kind)
        _CACHE[key] = Operands(L, N, K, exact, seed_of(preset, kind, exact))
    return _CACHE[key]


def gemm_run(L, P, A, sa, fp8, M, epi, bn, bias):
    """one oa_k_prefill_gemm call on A (P.a_operand): (rc, the BLOCK_N used, out with PAD sentinel rows)"""
    N, K = P.B.shape
    B, sb = (P.B8, P.sb) if fp8 else (P.B, None)
    if epi == 1:
        out = P.resid[:M + PAD].clone()
    else:
        out = torch.full((M + PAD, N // 2 if epi == 2 else N), float("nan"), dtype=BF16, device=dev())
    used = C.c_int32(-1)
    rc = L.oa_k_prefill_gemm(ptr(A), ptr(sa), ptr(B), ptr(sb), A_ROWS, M, N, K, epi, bn, ptr(out), ptr(bias), C.byref(used), None)
    return rc, used.value, out


def swiglu_split(acc, N):
    r = acc.view(acc.shape[0], N // 32, 2, 16)             # physical columns: 16 gate, then 16 up per 32
    return r[:, :, 0].reshape(acc.shape[0], N // 2), r[:, :, 1].reshape(acc.shape[0], N // 2)


def gemm_check(P, fp8, M, epi, bias, out, what, min_equal):
    N = P.B.shape[0]
    acc = (P.acc8 if fp8 else P.acc)[:M]
    tol = P.tol8 if fp8 else P.tol
    # rows past M: the NaN sentinels (store, SwiGLU) or the untouched residual rows
    tail = P.resid[M:M + PAD] if epi == 1 else None
    if epi == 1:
        assert same(out[M:], tail), f"{what}: a row >= M changed"
    else:
        assert (out[M:].view(torch.int16) == BF16_NAN).all(), f"{what}: a row >= M was written"
    if epi == 2:
        gte, up = swiglu_split(acc, N)
        ref = gte / (1 + torch.exp(-gte)) * up
        if P.exact:
            check_bf16(out[:M], ref, f"{what}", min_equal=0.0)        # exact g, u: within 1 ulp of fp64 silu(g) * u
        else:
            check_bf16(out[:M], ref, what, abs_tol=5 * tol, min_equal=min_equal)
        return
    ref = acc + (P.resid[:M].double() if epi == 1 else (bias.double() if bias is not None else 0.0))
    if P.exact:
        assert same(out[:M], ref.to(BF16)), f"{what}: {int((out[:M] != ref.to(BF16)).sum())} outputs differ from bf16(exact)"
    else:
        check_bf16(out[:M], ref, what, abs_tol=tol, min_equal=min_equal)


def gemm_variants(L, sms, M, N, fp8):
    """(block_n, persistent threshold or None) of each run at this M: the engine's choice, and every other BN at OTHER_BN_MS; a run at
    BN 128 goes once through the persistent kernel (threshold 1) and once through the tile kernel (threshold above any tile count)"""
    eng = pick_bn(L, M, N, sms, fp8)
    bns = [0] + ([b for b in BNS[fp8] if b != eng] if M in OTHER_BN_MS else [])
    runs = []
    for b in bns:
        if (b or eng) == 128:
            runs += [(b, "1"), (b, "1000000000")]
        else:
            runs.append((b, None))
    return eng, runs


ENGINE_BN = {}               # (preset, kind, M, fp8) -> the BLOCK_N the engine chose, recorded by test_projection


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("preset", PRESETS)
def test_projection(L, sms, monkeypatch, preset, kind):
    N, K = proj_shape(preset, kind)
    epi = KINDS[kind]
    use_bias = kind == "qkv" and PRESETS[preset][5]
    for exact in (True, False):
        P = operands(L, preset, kind, exact)
        bias = P.bias if use_bias else None
        for fp8 in (False, True):
            min_equal = MIN_EQUAL_FP8 if fp8 else (MIN_EQUAL if K <= 16384 else MIN_EQUAL_LONG_K)
            for M in MS + (MS_FP8 if fp8 else []):
                eng, runs = gemm_variants(L, sms, M, N, fp8)
                A, sa = P.a_operand(fp8, M)
                for bn, thr in runs:
                    if thr is None:
                        monkeypatch.delenv("OA_GEMM_PERSISTENT_MIN_TILES", raising=False)
                    else:
                        monkeypatch.setenv("OA_GEMM_PERSISTENT_MIN_TILES", thr)
                    kernel = "" if thr is None else (" persistent" if thr == "1" else " tile")
                    tag = f"{'exact' if exact else 'random'}{'/fp8' if fp8 else ''}"
                    what = f"{tag}: {preset} {kind} M {M} bn {bn or eng}{' (engine)' if bn == 0 else ''}{kernel}"
                    rc, used, out = gemm_run(L, P, A, sa, fp8, M, epi, bn, bias)
                    assert rc == 0, (what, rc, _lib.last_error())
                    assert used == (bn or eng), (what, used)
                    if bn == 0:
                        ENGINE_BN[preset, kind, M, fp8] = used
                    gemm_check(P, fp8, M, epi, bias, out, what, min_equal)
    monkeypatch.delenv("OA_GEMM_PERSISTENT_MIN_TILES", raising=False)
    report(f"{preset} {kind}")


def test_engine_block_n_choices_cover_32_64_128(L, sms):
    """the engine's BLOCK_N over the projection parametrization includes 32, 64 and 128, so none of them goes untested at a production K"""
    chosen = {pick_bn(L, M, proj_shape(p, k)[0], sms, fp8) for p in PRESETS for k in KINDS for fp8 in (False, True)
              for M in MS + (MS_FP8 if fp8 else [])}
    assert {32, 64, 128} <= chosen, chosen
    for key, bn in ENGINE_BN.items():       # what the entry point reported equals the host function
        assert bn == pick_bn(L, key[2], proj_shape(key[0], key[1])[0], sms, key[3]), key


# ------------------------------------------------------------------------------------------------ attention
# (pos0, new rows) of each prefill sequence: fresh prompts around the tile and page sizes, and continuations starting mid-page, one of
# them a single row after 16383 cached tokens.  pos0 = 1 (mod 64) puts the last query row of a warpgroup on the first key of a page: the
# boundary of the kernel's "does this warpgroup see this page" test.
FRESH = [(0, n) for n in (1, 63, 64, 65, 127, 128, 129, 1536, 8192)]
CONT = [(100, 28), (100, 300), (1540, 1), (1540, 700), (4095, 1), (4095, 129), (4095, 2000), (12000, 385), (16383, 1), (1, 127), (4033, 300)]
SEQS = FRESH + CONT
HEADS = [(32, 8, 64), (32, 8, 128), (40, 8, 128), (64, 8, 128),
         (10, 2, 128), (8, 1, 128)]     # one tensor-parallel rank of Qwen2.5-32B at t = 4 and of Llama-3-70B at t = 8
N_DECODE = [1, 37, 128]
LARGE_POOL = {False: 10000, True: 20000}     # pages of the 32/8/128 cache: more than 2 GiB, so byte offsets pass 2^31


class Batch:
    """the prefill sequences SEQS on one paged cache: random distinct pages from the top of the pool, host block tables"""

    def __init__(self, nh, nkv, D, fp8, seed):
        self.nh, self.nkv, self.D, self.fp8 = nh, nkv, D, fp8
        self.ctx = [p + n for p, n in SEQS]
        self.qlen = [n for _, n in SEQS]
        self.T = sum(self.qlen)
        self.maxp = MAX_POS // 64
        need = sum((c + 63) // 64 for c in self.ctx)
        self.num_pages = LARGE_POOL[fp8] if (nh, D) == (32, 128) else need + 50
        g = torch.Generator(device="cpu").manual_seed(seed)
        top = self.num_pages - need - 8 + torch.randperm(need + 8, generator=g)[:need]
        self.bt = np.zeros((len(SEQS), self.maxp), np.int32)
        k = 0
        for i, c in enumerate(self.ctx):
            n = (c + 63) // 64
            self.bt[i, :n] = top[k:k + n].numpy(); k += n
        # every cached token's (page, offset), concatenated over the sequences
        pages, offs = [], []
        for i, c in enumerate(self.ctx):
            t = np.arange(c)
            pages.append(self.bt[i, t // 64]); offs.append(t % 64)
        self.page = torch.from_numpy(np.concatenate(pages)).long().to(dev())
        self.off = torch.from_numpy(np.concatenate(offs)).long().to(dev())
        self.tok0 = np.concatenate([[0], np.cumsum(self.ctx)])           # first token of sequence i in the concatenation
        self.row0 = np.concatenate([[0], np.cumsum(self.qlen)])

    def cache(self, K, V, fill):
        """a cache whose cached tokens hold K, V [tokens, nkv, D] (bf16 values, or e4m3 bytes as uint8) and every other slot `fill`"""
        P, nkv, D = self.num_pages, self.nkv, self.D
        if self.fp8:
            c = torch.full((2, P, nkv, 64 * D), fill, dtype=torch.uint8, device=dev())
            c[0].view(P, nkv, 64, D).permute(0, 2, 1, 3)[self.page, self.off] = K
            c[1].view(P, nkv, D, 64).permute(0, 3, 1, 2)[self.page, self.off] = V
        else:
            c = torch.full((2, P, nkv, 64, D), fill, dtype=BF16, device=dev())
            c[0].permute(0, 2, 1, 3)[self.page, self.off] = K
            c[1].permute(0, 2, 1, 3)[self.page, self.off] = V
        return c


def step_attention(L, B, q, cache, ks, vs, n_decode=0, dec_ctx=None, dec_bt=None, prefill=True):
    """oa_k_step_attention on n_decode decode sequences (ctx dec_ctx, block tables dec_bt) followed by B's prefill sequences (if prefill).
    Returns out [rows + PAD, nh * D] (PAD NaN sentinel rows after the last row)."""
    ctx = list(dec_ctx or []) + (B.ctx if prefill else [])
    ql = [1] * n_decode + (B.qlen if prefill else [])
    bt = np.ascontiguousarray(np.concatenate(([dec_bt] if n_decode else []) + ([B.bt] if prefill else [])).astype(np.int32))
    ctx_a, ql_a = np.array(ctx, np.int32), np.array(ql, np.int32)
    rows = int(ql_a.sum())
    out = torch.full((rows + PAD, B.nh * B.D), float("nan"), dtype=BF16, device=dev())
    rc = L.oa_k_step_attention(ptr(q), ptr(out), ptr(cache), B.num_pages, bt.ctypes.data, B.maxp, ctx_a.ctypes.data, ql_a.ctypes.data,
                               len(ctx), n_decode, B.nh, B.nkv, B.D, ks if B.fp8 else 0.0, vs if B.fp8 else 0.0, None)
    assert rc == 0, (rc, _lib.last_error())
    assert (out[rows:].view(torch.int16) == BF16_NAN).all(), "a row after the last one was written"
    return out[:rows]


def qpos_of(B):
    return torch.from_numpy(np.concatenate([np.arange(p, p + n) for p, n in SEQS])).long().to(dev())


def seq_of_row(B):
    return torch.from_numpy(np.repeat(np.arange(len(SEQS)), B.qlen)).long().to(dev())


def test_prefill_attention_indicator_exact(L):
    """Q = 0: every visible key has weight exactly 1 and l = qpos + 1.  V[t, d] = 1 where d = chunk(t) mod D: each output element is
    (visible keys of its chunks) / l, computed in fp32 as the kernel does (1/l, or v_scale/l, then one product) and compared bit for bit"""
    for nh, nkv, D in HEADS:
        for fp8 in (False, True):
            B = Batch(nh, nkv, D, fp8, seed_of("ind", nh, D, fp8))
            tok = torch.cat([torch.arange(c, device=dev()) for c in B.ctx])
            onehot = ((tok // 64) % D)[:, None] == torch.arange(D, device=dev())[None, :]
            vs = 0.5
            if fp8:
                one = torch.tensor([1.0]).to(FP8).view(torch.uint8).item()
                V = (onehot.to(torch.uint8) * one)[:, None, :].expand(-1, nkv, -1)
                K = torch.zeros_like(V)
            else:
                V = onehot.to(BF16)[:, None, :].expand(-1, nkv, -1)
                K = torch.zeros_like(V)
            cache = B.cache(K, V, 0)
            q = torch.zeros(B.T, nh * D, dtype=BF16, device=dev())
            out = step_attention(L, B, q, cache, 1.0, vs)
            qpos = qpos_of(B)
            # count[r, d] = #{t <= qpos : (t // 64) % D == d}
            full, rem = (qpos + 1) // 64, (qpos + 1) % 64           # full chunks, then rem keys of chunk `full`
            d = torch.arange(D, device=dev())[None, :]
            cnt = (64 * ((full[:, None] - d + D - 1).clamp_min(0) // D)).float()
            cnt += torch.where((full % D)[:, None] == d, rem[:, None].float(), 0.0)
            inv = (torch.tensor(vs if fp8 else 1.0, dtype=torch.float32, device=dev()) / (qpos + 1).float())[:, None]
            ref = (cnt * inv).to(BF16)
            got = out.view(B.T, nh, D)
            bad = got != ref[:, None, :]
            assert not bad.any(), f"{nh}/{nkv}/{D} fp8 {fp8}: {int(bad.sum())} outputs differ, e.g. row {int(bad.nonzero()[0][0])}"


def needle_cache(B, sign, seed):
    """K encodes each key's position t in base-256 (bf16) or base-16 (e4m3) digits, Q = sign * c * (the digit weights), so that q.k = sign
    * c * t exactly; V[t, kvh, :] random in [1, 2) on the 7-bit (bf16) or 3-bit (e4m3) grid.  Returns (q, cache, V as bf16 values)."""
    nkv, D = B.nkv, B.D
    g = torch.Generator(device="cpu").manual_seed(seed)
    tok = torch.cat([torch.arange(c) for c in B.ctx]).to(dev())
    n = tok.numel()
    base, nd = (16, 4) if B.fp8 else (256, 2)
    digits = torch.stack([(tok // base ** i) % base for i in range(nd)], 1).float()
    Kf = torch.zeros(n, nkv, D, device=dev())
    Kf[:, :, :nd] = digits[:, None, :]
    steps = 8 if B.fp8 else 128
    Vf = 1 + torch.randint(0, steps, (n, nkv, D), generator=g).float().to(dev()) / steps
    c = 128.0
    qrow = torch.zeros(D)
    qrow[:nd] = sign * c * torch.tensor([float(base ** i) for i in range(nd)])
    q = qrow.to(BF16).to(dev())[None, :].repeat(B.T, B.nh)
    if B.fp8:
        cache = B.cache(Kf.to(FP8).view(torch.uint8), Vf.to(FP8).view(torch.uint8), 0)
    else:
        cache = B.cache(Kf.to(BF16), Vf.to(BF16), 0)
    return q, cache, Vf.to(BF16)


def test_prefill_attention_needle_exact(L):
    """each row attends only its own position (c > 0) or only position 0 (c < 0): its output is that key's V bit for bit.  Checks the
    page lookup, pos0, the head -> kv-head map and the output row."""
    for nh, nkv, D in HEADS:
        for fp8 in (False, True):
            B = Batch(nh, nkv, D, fp8, seed_of("needle", nh, D, fp8))
            qpos, seq = qpos_of(B), seq_of_row(B)
            kvh = torch.arange(nh, device=dev()) // (nh // nkv)
            tok0 = torch.from_numpy(B.tok0[:-1]).long().to(dev())
            for sign in (1, -1):
                q, cache, V = needle_cache(B, sign, seed_of("needle-v", nh, D, fp8))
                vs = 2.0 if fp8 else 1.0
                out = step_attention(L, B, q, cache, 1.0, vs).view(B.T, nh, D)
                t = tok0[seq] + (qpos if sign > 0 else 0)
                ref = (V[t][:, kvh, :].float() * vs).to(BF16)
                bad = out != ref
                assert not bad.any(), f"{nh}/{nkv}/{D} fp8 {fp8} sign {sign}: {int(bad.sum())} outputs differ, e.g. row {int(bad.nonzero()[0][0])}"


def attn_ref64(B, q, K, V):
    """fp64 causal attention of every row of B over its sequence's tokens; K, V [tokens, nkv, D] (fp64 values)"""
    nh, nkv, D = B.nh, B.nkv, B.D
    grp = nh // nkv
    out = torch.empty(B.T, nh, D, dtype=torch.float64, device=dev())
    for i, (p0, n) in enumerate(SEQS):
        k = K[B.tok0[i]:B.tok0[i + 1]].repeat_interleave(grp, 1)     # [ctx, nh, D]
        v = V[B.tok0[i]:B.tok0[i + 1]].repeat_interleave(grp, 1)
        for r in range(0, n, 256):
            rr = min(n, r + 256)
            qq = q[B.row0[i] + r:B.row0[i] + rr].view(rr - r, nh, D).double()
            s = torch.einsum("rhd,khd->hrk", qq, k) / D ** 0.5
            pos = torch.arange(p0 + r, p0 + rr, device=dev())[:, None]
            s.masked_fill_(torch.arange(k.shape[0], device=dev())[None, :] > pos, float("-inf"))
            out[B.row0[i] + r:B.row0[i] + rr] = torch.einsum("hrk,khd->rhd", torch.softmax(s, -1), v)
    return out


def test_prefill_attention_random_stale_tails_and_mixed_steps(L):
    """random Q, K, V against fp64 (bound relative to each row's rms); junk in every slot past the contexts changes no bit; in a mixed
    step the decode rows equal a decode-only launch and the prefill rows a prefill-only launch, bit for bit"""
    worst = {}
    for nh, nkv, D in HEADS:
        for fp8 in (False, True):
            B = Batch(nh, nkv, D, fp8, seed_of("rand", nh, D, fp8))
            g = torch.Generator(device="cpu").manual_seed(seed_of("rand-data", nh, D, fp8))
            n = int(B.tok0[-1])
            Kr = torch.randn(n, nkv, D, generator=g).to(dev())
            Vr = torch.randn(n, nkv, D, generator=g).to(dev())
            q = torch.randn(B.T, nh * D, generator=g).to(BF16).to(dev())
            if fp8:
                ks, vs = 0.37, 2.9
                K8, V8 = (2 * Kr).to(FP8), Vr.to(FP8)
                Kd, Vd = K8.double() * ks, V8.double() * vs
                K, V = K8.view(torch.uint8), V8.view(torch.uint8)
                junk = 0x7E                                   # e4m3 448: large and finite
            else:
                ks = vs = 0.0
                K, V = Kr.to(BF16), Vr.to(BF16)
                Kd, Vd = K.double(), V.double()
                junk = JUNK
            cache0 = B.cache(K, V, 0)
            out = step_attention(L, B, q, cache0, ks, vs)
            ref = attn_ref64(B, q, Kd, Vd)
            rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
            err = ((out.view(B.T, nh, D).double() - ref).abs() / rms).max().item()
            worst[nh, D, fp8] = err
            assert err < ATTN_REL_TOL, f"{nh}/{nkv}/{D} fp8 {fp8}: error {err:.3e} of the row rms"
            del ref, rms
            # stale tails: every slot outside the contexts holds large finite junk
            cachej = B.cache(K, V, junk)
            assert same(step_attention(L, B, q, cachej, ks, vs), out), f"{nh}/{nkv}/{D} fp8 {fp8}: junk past the contexts changed the output"
            del cachej
            # mixed steps: n_decode single-row sequences (on the prefill sequences' pages) ahead of the prefill rows
            rng = np.random.default_rng(seed_of("mixed", nh, D, fp8))
            for nd in N_DECODE:
                src = rng.integers(0, len(SEQS), nd)
                dctx = [int(rng.integers(1, B.ctx[s] + 1)) for s in src]
                dbt = B.bt[src]
                qd = torch.randn(nd, nh * D, generator=g).to(BF16).to(dev())
                mixed = step_attention(L, B, torch.cat([qd, q]), cache0, ks, vs, nd, dctx, dbt)
                dec = step_attention(L, B, qd, cache0, ks, vs, nd, dctx, dbt, prefill=False)
                assert same(mixed[:nd], dec), f"{nh}/{nkv}/{D} fp8 {fp8} n_decode {nd}: decode rows differ from a decode-only launch"
                assert same(mixed[nd:], out), f"{nh}/{nkv}/{D} fp8 {fp8} n_decode {nd}: prefill rows differ from a prefill-only launch"
            del cache0
            torch.cuda.empty_cache()
    print("\nattention on random data, largest error over the row rms: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ------------------------------------------------------------------------------------------------ the prefill KV writer on a > 2 GiB pool
def rope_tables(D, theta=500000.0):
    half = D // 2
    inv = theta ** (-2.0 * torch.arange(half, dtype=torch.float64) / D)
    a = torch.arange(MAX_POS, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.cos(a).float().to(dev()).contiguous(), torch.sin(a).float().to(dev()).contiguous()


def q8(x, scale):
    """the byte an fp8 writer stores for x (fp32 math): e4m3(x * (1/scale)), saturating"""
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(scale, dtype=torch.float32)
    return (x.float() * inv.to(x.device)).clamp(-448, 448).to(FP8)


@pytest.mark.parametrize("fp8", [False, True])
def test_kv_write_large_pool(L, fp8):
    nh, nkv, D = 32, 8, 128
    T, P = 8192, LARGE_POOL[fp8]
    g = torch.Generator(device="cpu").manual_seed(11 + fp8)
    # positions: a 4096-token chunk continuing at 12288, then 4096 scattered positions over [0, 16384)
    pos = torch.cat([torch.arange(12288, 16384), torch.randint(0, MAX_POS, (T - 4096,), generator=g)]).to(torch.int32)
    top = torch.arange(P - 64, P)                                  # the pool's top pages, then random slots anywhere
    slots = torch.cat([(top[:, None] * 64 + torch.arange(64)[None, :]).flatten(), torch.randperm(P * 64 - 4096, generator=g)[:T - 4096]])
    slots = slots[torch.randperm(T, generator=g)].to(torch.int32)
    pos, slots = pos.to(dev()), slots.to(dev())
    qkv = (torch.randn(T, (nh + 2 * nkv) * D, generator=g) * 3).to(BF16).to(dev())
    cos, sin = rope_tables(D)
    q_out = torch.full((T + PAD, nh * D), float("nan"), dtype=BF16, device=dev())
    fill = 0x7F if fp8 else 0x7F7F                                  # an e4m3 NaN code / a bf16 value no writer produces
    ks, vs = 0.37, 2.9
    if fp8:
        cache = torch.full((2, P, nkv, 64 * D), fill, dtype=torch.uint8, device=dev())
        rc = L.oa_k_kv_write_fp8(ptr(qkv), ptr(pos), ptr(slots), ptr(cos), ptr(sin), ptr(q_out), ptr(cache), P, T, nh, nkv, D, ks, vs, None)
    else:
        cache = torch.full((2, P, nkv, 64, D), fill, dtype=torch.int16, device=dev()).view(BF16)
        rc = L.oa_k_kv_write(ptr(qkv), ptr(pos), ptr(slots), ptr(cos), ptr(sin), ptr(q_out), ptr(cache), P, T, nh, nkv, D, None)
    assert rc == 0, _lib.last_error()
    assert cache.numel() * cache.element_size() > 2 ** 31
    # fp64 RoPE of the bf16 q and k
    x = qkv.double().view(T, nh + 2 * nkv, D)
    c, s = cos[pos.long()].double()[:, None, :], sin[pos.long()].double()[:, None, :]
    lo, hi = x[:, :nh + nkv, :D // 2], x[:, :nh + nkv, D // 2:]
    rot = torch.cat([lo * c - hi * s, hi * c + lo * s], -1)
    tol = 2.0 ** -20 * qkv.float().abs().max().item()            # the fp32 rotation's error where lo * c - hi * s cancels
    check_bf16(q_out[:T].view(T, nh, D), rot[:, :nh], "q: kv write", abs_tol=tol)
    assert (q_out[T:].view(torch.int16) == BF16_NAN).all()
    page, off = slots.long() // 64, slots.long() % 64
    raw = cache if fp8 else cache.view(torch.int16)
    if fp8:
        k = cache[0].view(P, nkv, 64, D)[page, :, off]
        v = cache[1].view(P, nkv, D, 64)[page, :, :, off]
        kr = rot[:, nh:]
        u = torch.maximum(ulp(kr), torch.full_like(kr, tol))       # the kernel's bf16 k lies within this of the fp64 rotation
        g8 = k.view(FP8).double()
        assert ((g8 >= q8((kr - u).to(BF16), ks).double()) & (g8 <= q8((kr + u).to(BF16), ks).double())).all(), "k8 outside its interval"
        assert torch.equal(v, q8(x[:, nh + nkv:].to(BF16), vs).view(torch.uint8)), "v8 bytes"
        written = torch.zeros(P, 64, dtype=torch.bool, device=dev())
        written[page, off] = True
        kk = raw[0].view(P, nkv, 64, D).permute(0, 2, 1, 3)
        vv = raw[1].view(P, nkv, D, 64).permute(0, 3, 1, 2)
    else:
        k = cache[0].permute(0, 2, 1, 3)[page, off]
        v = cache[1].permute(0, 2, 1, 3)[page, off]
        check_bf16(k, rot[:, nh:], "k: kv write", abs_tol=tol)
        assert torch.equal(v, qkv.view(T, nh + 2 * nkv, D)[:, nh + nkv:]), "V is copied bit for bit"
        written = torch.zeros(P, 64, dtype=torch.bool, device=dev())
        written[page, off] = True
        kk = raw[0].permute(0, 2, 1, 3)
        vv = raw[1].permute(0, 2, 1, 3)
    assert (kk[~written] == fill).all() and (vv[~written] == fill).all(), "a KV row outside `slots` changed"
    report(f"kv write fp8 {fp8}")


# ------------------------------------------------------------------------------------------------ glue
@pytest.mark.parametrize("H", [2048, 4096, 5120, 8192])
def test_rmsnorm_production_shapes(L, H):
    for T in (1623, 8192):
        g = gen(seed_of("rms", H, T))
        x = (torch.randn(T, H, device=dev(), generator=g) * (1 + 3 * torch.rand(T, 1, device=dev(), generator=g))).to(BF16)
        gain = (1 + 0.3 * torch.randn(H, device=dev(), generator=g)).to(BF16)
        y = torch.full((T + PAD, H), float("nan"), dtype=BF16, device=dev())
        assert L.oa_k_rmsnorm(ptr(x), ptr(gain), ptr(y), T, H, EPS, None) == 0
        torch.cuda.synchronize()
        xd = x.double()
        ref = xd * torch.rsqrt((xd * xd).mean(1, keepdim=True) + EPS) * gain.double()
        check_bf16(y[:T], ref, f"rmsnorm: T {T} H {H}", min_equal=0.999)      # measured 0.99999
        assert (y[T:].view(torch.int16) == BF16_NAN).all()
    report(f"rmsnorm H {H}")


@pytest.mark.parametrize("vocab,H", [(152064, 5120), (128256, 8192)])
def test_embed_gather(L, vocab, H):
    T = 8192
    g = gen(vocab)
    table = torch.randn(vocab, H, device=dev(), generator=g).to(BF16)
    ids = torch.randint(0, vocab, (T,), device=dev(), generator=g, dtype=torch.int32)
    top = vocab - 1 - torch.randint(0, vocab // 100, (T // 4,), device=dev(), generator=g, dtype=torch.int32)   # the top 1% of rows
    ids[::4] = top
    ids[1:50:7] = -1
    ids[2:50:7] = vocab
    ids[3:50:7] = vocab - 1
    ids[4:50:7] = -2 ** 31
    ids[5:50:7] = 2 ** 31 - 1
    out = torch.full((T + PAD, H), float("nan"), dtype=BF16, device=dev())
    assert L.oa_k_embed_gather(ptr(ids), ptr(table), ptr(out), T, H, vocab, None) == 0
    idx = torch.where((ids < 0) | (ids >= vocab), 0, ids).long()       # ids outside [0, vocab) read row 0
    assert same(out[:T], table[idx])
    assert (out[T:].view(torch.int16) == BF16_NAN).all()


@pytest.mark.parametrize("V,K", [(128256, 2048), (152064, 5120)])
def test_masked_argmax_prefill_rows(L, sms, V, K):
    """the LM head over the sampled rows of a prefill step (M > 128), at the BLOCK_N pick_bn chooses; masks and ties as in the decode
    file's test_masked_argmax"""
    words = (V + 31) // 32
    for M in (129, 2048):
        bn = pick_bn(L, M, V, sms, False)
        g = torch.Generator(device="cpu").manual_seed(V + M)
        A = torch.randn(M, K, generator=g).to(BF16)
        B = (torch.randn(V, K, generator=g) * 0.1).to(BF16)
        j1, j2, j3 = 3 * V // 10, V - 300, V // 2 + 5
        B[j2] = B[j1]; B[j3 + 1] = B[j3]                          # exact ties: across tiles, and inside one 32-column chunk
        A, B = A.to(dev()), B.to(dev())
        bits = np.zeros((6, words * 32), np.bool_)
        rng = np.random.default_rng(V + M)
        bits[0] = rng.random(words * 32) < 0.3
        bits[1, V - 1] = True
        w = (V // 3 // 32 + 1) * 32
        bits[2, w - 3:w + 2] = True
        bits[2, 40] = True
        bits[4, [j1, j2]] = True
        bits[5, [j3, j3 + 1]] = True
        bits[:, V:] = False
        table = torch.from_numpy(np.packbits(bits, axis=1, bitorder="little").view(np.int32).copy()).to(dev())
        slot = torch.from_numpy(rng.integers(-1, 6, M).astype(np.int32)).to(dev())
        slot[:12] = torch.tensor([-1, 0, 1, 2, 3, 4, 5, -1, 0, 2, 1, 4], dtype=torch.int32)
        logits = torch.full((M, V), float("nan"), dtype=torch.float32, device=dev())
        ids = torch.full((M,), -1, dtype=torch.int32, device=dev())
        rc = L.oa_k_gemm_logits_masked(ptr(A), ptr(B), M, V, K, bn, ptr(table), ptr(slot), words, 0, ptr(logits), ptr(ids), None)
        assert rc == 0, _lib.last_error()
        ref = A.double() @ B.double().T
        assert ((logits.double() - ref).abs() <= 1e-4 * K ** 0.5 + 1e-5 * ref.abs()).all(), (M, bn)
        assert torch.equal(logits[:, j1], logits[:, j2]) and torch.equal(logits[:, j3], logits[:, j3 + 1])
        allowed = torch.from_numpy(bits[:, :V].copy()).to(dev())
        ok = torch.ones(M, V, dtype=torch.bool, device=dev())
        masked = slot >= 0
        ok[masked] = allowed[slot[masked].long()]
        lg = torch.where(ok, logits, torch.tensor(-float("inf"), device=dev()))
        mx = lg.max(1, keepdim=True).values
        first = torch.where(ok & (lg == mx), torch.arange(V, device=dev())[None, :], V).min(1).values
        exp = torch.where(first == V, 0, first)                    # a row allowing nothing takes id 0
        assert torch.equal(ids.long(), exp), (M, bn)
        assert ids[2].item() == V - 1 and ids[4].item() == 0 and ids[5].item() == j1 and ids[11].item() == j1 and ids[6].item() == j3
