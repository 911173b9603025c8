"""The tensor-parallel collectives of DeviceModel::forward at the TP presets' per-rank shapes, on one GPU (pytest -m gpu): the decode o / down
finish (stream-K partial -> "buffer written" signal -> rank-ordered all-reduce fused with the residual add and RMSNorm), the prefill
all-reduce (one-shot, and two-shot: reduce-scatter + all-gather) and the vocab-parallel greedy arg-max.

Every collective reaches its peers through a device table of pointers.  The C entry points (oa_k_tp_*) point the t entries at t local buffers
and launch each rank's kernels in turn on one stream, so each kernel does exactly what rank r does on t GPUs; only the memory behind the
pointers is local instead of NVLink-mapped.  No barrier kernel runs: the decode entry point reads the flags back and launches the waiting
consumers only once every signal is there, and stream order stands in for the prefill path's barriers.

The all-reduces are compared bit for bit with a torch float32 emulation of the kernels' sum (IEEE adds, in rank order from a zero
accumulator, then the residual), on data where another order changes bits, and end to end with fp64.  The arg-max is compared with the
kernel's own logits, ties and empty grammar masks included, and the logits with fp64.

Bounds and exact-match floors: tests/kernel_ref.py, and the floor for bf16 partials below.  Measured on an H100 80GB HBM3 (SXM, 132 SMs)
at its 700 W default power limit, where the file runs in about 20 s.  Smallest exact-match fractions of x against bf16(fp64) over every
case, M, BLOCK_N and CTA count: fp32 partials 0.9944 (down of Llama-3-8B t = 2), bf16 partials 0.6504 (each rank's partial is rounded to
bf16 before the sum); xn against the fp64 norm of the kernel's own x: 0.9998.  Outputs that the residual-first order changes: 1e-5 to 3e-5
of the decode rows, enough to catch a reordered sum."""
import ctypes as C
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from opsagent_b200 import _lib  # noqa: E402
from kernel_ref import ACC_TOL_BF16_PER_K, BF16, MATCH, MIN_EQUAL, MIN_EQUAL_LONG_K, check_bf16, dev, ptr, report, same  # noqa: E402

BF16_NAN, F32_NAN = 0x7FC0, 0x7FC00000     # output sentinels: what the kernels must not write keeps these bits
FLAG_FILL = 0x5A5A5A5A                      # flag sentinel: equal to no epoch used below
EPS = 1e-5
MAXM = 256
MS = [1, 5, 64, 128, 129, 256]
MIN_EQUAL_BF16_PARTIALS = 0.6              # x on bf16 partials: every rank's partial carries its own bf16 rounding

# name: (hidden, n_heads, n_kv, head_dim, ffn, vocab, t) of the tensor-parallel presets (csrc/config.hpp); one rank holds n_heads / t heads,
# ffn / t of the ffn and vocab / t of the vocabulary
CASES = {
    "llama-3-8b/tp2": (4096, 32, 8, 128, 14336, 128256, 2),
    "qwen2.5-32b/tp4": (5120, 40, 8, 128, 27648, 152064, 4),
    "qwen2.5-32b/tp8": (5120, 40, 8, 128, 27648, 152064, 8),
    "llama-3-70b/tp8": (8192, 64, 8, 128, 28672, 128256, 8),
}


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


def parr(ts):
    """a host array of the tensors' device pointers (None: a null array)"""
    return None if ts is None else (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32)


def rank_ordered(x0, parts, order):
    """bf16(x0 + sum of the partials in `order`, from a zero accumulator), in fp32 as the all-reduce kernels add"""
    acc = torch.zeros(x0.shape, dtype=torch.float32, device=dev())
    for r in order:
        acc = acc + parts[r].float()
    return (x0.float() + acc).to(BF16)


def residual_first(x0, parts):
    """the same sum in another order: the residual first, then the ranks in reverse (for t = 2 the reversed rank sum alone is the same)"""
    acc = x0.float()
    for p in reversed(parts):
        acc = acc + p.float()
    return acc.to(BF16)


# ------------------------------------------------------------------------------------------------ decode: o / down finish on t ranks
class RowPar:
    """One row-parallel projection of a case: A [MAXM, K] and B [H, K] cut by columns into t rank shards A[r] [MAXM, K/t], B[r] [H, K/t], so
    that the shards' products sum to the full product.  acc[r]: fp64 A[r].B[r]^T."""

    def __init__(self, case, kind):
        H, nh, nkv, D, F, V, t = CASES[case]
        K = nh * D if kind == "o" else F
        self.H, self.K, self.t, self.kr = H, K, t, K // t
        g = gen(seed_of(case, kind))
        A = torch.randn(MAXM, K, device=dev(), generator=g).to(BF16)
        B = (torch.randn(H, K, device=dev(), generator=g) * K ** -0.5).to(BF16)
        kr = self.kr
        self.A = [A[:, r * kr:(r + 1) * kr].contiguous() for r in range(t)]
        self.B = [B[:, r * kr:(r + 1) * kr].contiguous() for r in range(t)]
        del A, B
        self.acc = [a.double() @ b.double().T for a, b in zip(self.A, self.B)]
        self.full = sum(self.acc)
        self.tol_r = [ACC_TOL_BF16_PER_K * kr * a.pow(2).mean().sqrt().item() for a in self.acc]
        self.tol = ACC_TOL_BF16_PER_K * K * self.full.pow(2).mean().sqrt().item()
        self.min_equal = MIN_EQUAL if K <= 16384 else MIN_EQUAL_LONG_K
        g = gen(seed_of(case, kind, "x"))
        self.x0 = torch.randn(MAXM, H, device=dev(), generator=g).to(BF16)
        self.gain = (1 + 0.3 * torch.randn(H, device=dev(), generator=g)).to(BF16)


def new_flags():
    return torch.full((8, 8), FLAG_FILL, dtype=torch.int32, device=dev())


def check_flags(flags, t, epoch, what):
    f = flags.cpu().numpy().view(np.uint32)
    assert (f[:t, :t] == np.uint32(epoch)).all(), f"{what}: flags {f[:t, :t].tolist()} != epoch {epoch:#x}"
    assert (f[t:] == FLAG_FILL).all() and (f[:, t:] == FLAG_FILL).all(), f"{what}: a flag outside [t][t] changed"


def rp_run(L, P, M, bn, G, bf16p, x0, flags=None, epoch=1, launches=1):
    """oa_k_tp_row_parallel with every rank's x = x0 and NaN partials / xn: (rc, partials, x, xn, flags)"""
    parts = [torch.full((MAXM, P.H), float("nan"), dtype=BF16 if bf16p else torch.float32, device=dev()) for _ in range(P.t)]
    xs = [x0.clone() for _ in range(P.t)]
    xns = [torch.full_like(x0, float("nan")) for _ in range(P.t)]
    flags = new_flags() if flags is None else flags
    rc = L.oa_k_tp_row_parallel(P.t, parr(P.A), parr(P.B), M, P.H, P.kr, bn, G, int(bf16p), parr(parts), parr(xs), parr(xns), ptr(P.gain), EPS,
                                ptr(flags), epoch, launches, None)
    return rc, parts, xs, xns, flags


def rp_configs(sms):
    """(M, block_n, n_ctas) the engine can run: two 128-row slots (M > 128) take block_n 128"""
    return [(M, bn, G) for M in MS for G in (sms, 7) for bn in ((64, 128, 256) if M <= 128 else (128,))]


@pytest.mark.parametrize("kind", ["o", "down"])
@pytest.mark.parametrize("case", CASES)
def test_row_parallel_all_reduce(L, sms, case, kind):
    P = RowPar(case, kind)
    t, H, x0 = P.t, P.H, P.x0
    reordered = compared = 0
    for M, bn, G in rp_configs(sms):
        parts32 = None
        for bf16p in (False, True):
            what = f"{case} {kind} M {M} bn {bn} n_ctas {G} {'bf16' if bf16p else 'fp32'} partials"
            rc, parts, xs, xns, flags = rp_run(L, P, M, bn, G, bf16p, x0)
            assert rc == 0, (what, rc, _lib.last_error())
            check_flags(flags, t, 1, what)
            # the partials: fp32 within the accumulation bound of fp64; bf16 = the fp32 partial rounded (both sum the CTA pieces in order)
            if not bf16p:
                parts32 = parts
                for r in range(t):
                    err = (parts[r][:M].double() - P.acc[r][:M]).abs() - 2.0 ** -23 * P.acc[r][:M].abs()
                    assert (err <= P.tol_r[r]).all(), f"partial of rank {r}: {what}: {err.max().item()} > {P.tol_r[r]}"
            else:
                for r in range(t):
                    assert same(parts[r][:M], parts32[r][:M].to(BF16)), f"bf16 partial of rank {r} vs the rounded fp32 one: {what}"
            for r in range(t):
                assert torch.equal(bits(parts[r][M:]), torch.full_like(bits(parts[r][M:]), BF16_NAN if bf16p else F32_NAN)), \
                    f"partial rows >= M of rank {r}: {what}"
            # the all-reduce: every rank holds bit for bit the rank-ordered fp32 sum
            ref = rank_ordered(x0[:M], [p[:M] for p in parts], range(t))
            for r in range(t):
                assert same(xs[r][:M], ref), f"x of rank {r} vs the rank-ordered sum: {what}"
                assert same(xs[r][M:], x0[M:]) and (xns[r][M:].view(torch.int16) == BF16_NAN).all(), f"x / xn rows >= M of rank {r}: {what}"
                if r:
                    assert same(xns[r], xns[0]), f"xn of rank {r} vs rank 0: {what}"
            reordered += int((bits(residual_first(x0[:M], [p[:M] for p in parts])) != bits(ref)).sum())
            compared += M * H
            # end to end against fp64: bf16 partials add their own rounding, at most 2^-8 |p| each
            exact = x0[:M].double() + P.full[:M]
            extra = sum(p[:M].double().abs() for p in parts) * 2.0 ** -8 if bf16p else torch.zeros_like(exact)
            tag = "/bf16 partials" if bf16p else ""
            check_bf16(xs[0][:M], exact, f"x{tag}: {what}", exact - extra, exact + extra, abs_tol=P.tol,
                       min_equal=MIN_EQUAL_BF16_PARTIALS if bf16p else P.min_equal)
            xk = xs[0][:M].double()
            check_bf16(xns[0][:M], xk * torch.rsqrt((xk * xk).mean(1, keepdim=True) + EPS) * P.gain.double(), f"xn{tag}: {what}")
            if G == 7 and bn == 128:                          # a second call on fresh buffers
                rc, parts2, xs2, xns2, _ = rp_run(L, P, M, bn, G, bf16p, x0)
                assert rc == 0 and all(same(a, b) for a, b in zip(parts + xs + xns, parts2 + xs2 + xns2)), f"second call: {what}"
    MATCH["x differing in the reordered sum"] = reordered / compared
    assert reordered > 0, f"{case} {kind}: the rank-order check cannot tell a reordered sum apart"
    report(f"{case} {kind}")


@pytest.mark.parametrize("bf16p", [False, True])
@pytest.mark.parametrize("case", ["llama-3-8b/tp2", "qwen2.5-32b/tp8"])
def test_row_parallel_handshake_across_the_epoch_wrap(L, sms, case, bf16p):
    """the signal flags show each launch's epoch through the uint32 wrap, the done counters re-arm between launches (a counter that did not
    would leave launch 2 unsignalled: the entry point returns an error), and three launches equal three rank-ordered sums in turn"""
    P = RowPar(case, "o")
    t, x0 = P.t, P.x0
    for M in (5, 129):
        what = f"{case} M {M} {'bf16' if bf16p else 'fp32'} partials"
        flags, x = new_flags(), x0
        for e in (0xFFFFFFFE, 0xFFFFFFFF, 0):                 # one launch per call, on one flags array
            rc, parts, xs, xns, flags = rp_run(L, P, M, 128, sms, bf16p, x, flags=flags, epoch=e)
            assert rc == 0, (what, e, _lib.last_error())
            check_flags(flags, t, e, f"{what} epoch {e:#x}")
            assert all(same(xs[r], xs[0]) for r in range(t))
            x, xn = xs[0], xns[0]
        rc, parts3, xs3, xns3, flags3 = rp_run(L, P, M, 128, sms, bf16p, x0, epoch=0xFFFFFFFE, launches=3)
        assert rc == 0, (what, _lib.last_error())
        check_flags(flags3, t, 0, f"{what} launches 3")
        exp = x0.clone()
        for _ in range(3):
            exp[:M] = rank_ordered(exp[:M], [p[:M] for p in parts3], range(t))
        for r in range(t):
            assert same(xs3[r], exp) and same(xs3[r], x) and same(xns3[r], xn), f"rank {r} after three launches: {what}"


# ------------------------------------------------------------------------------------------------ prefill: one-shot and two-shot all-reduce
PREFILL_T = [129, 1023, 1024, 8192]
# shapes the launchers accept that production never makes: fewer 16-byte vectors than ranks, or a count that t does not divide, so that
# the last two-shot slices are short or empty
SYNTHETIC = [(t, T, H) for t in (3, 5, 7) for T, H in ((1, 8), (3, 40), (257, 264))]
PAD = 2                                      # sentinel rows after T in x and gather


def prefill_partials(t, T, H, seed):
    """random bf16 partials where rank 0 and rank t-1 hold large cancelling values (2^8 .. 2^21) on half the elements: partial sums round
    at the large value's ulp, so the order of the adds changes bits"""
    g = gen(seed)
    parts = [torch.randn(T, H, device=dev(), generator=g).to(BF16) for _ in range(t)]
    big = torch.exp2(torch.randint(8, 21, (T, H), device=dev(), generator=g).float()) * (1 + torch.rand(T, H, device=dev(), generator=g))
    big = (big * torch.where(torch.rand(T, H, device=dev(), generator=g) < 0.5, -1.0, 1.0)).to(BF16)
    pair = torch.rand(T, H, device=dev(), generator=g) < 0.5
    parts[0] = torch.where(pair, big, parts[0])
    parts[-1] = torch.where(pair, -big, parts[-1])
    del big, pair
    x0 = torch.randn(T, H, device=dev(), generator=g).to(BF16)
    return parts, x0


def prefill_run(L, parts, x0, T, H, two_shot):
    t = len(parts)
    xs = []
    for _ in range(t):
        x = torch.full((T + PAD, H), float("nan"), dtype=BF16, device=dev())
        x[:T] = x0
        xs.append(x)
    gath = [torch.full((T + PAD, H), float("nan"), dtype=BF16, device=dev()) for _ in range(t)] if two_shot else None
    rc = L.oa_k_tp_allreduce_prefill(t, parr(parts), parr(xs), parr(gath), T, H, int(two_shot), None)
    return rc, xs, gath


def check_prefill(L, t, T, H, seed, what, must_reorder):
    parts, x0 = prefill_partials(t, T, H, seed)
    ref = rank_ordered(x0, parts, range(t))
    if must_reorder:
        assert (bits(residual_first(x0, parts)) != bits(ref)).any(), f"{what}: the rank-order check cannot tell a reordered sum apart"
    one = None
    for two_shot in (False, True):
        w = f"{what} {'two' if two_shot else 'one'}-shot"
        rc, xs, gath = prefill_run(L, parts, x0, T, H, two_shot)
        assert rc == 0, (w, rc, _lib.last_error())
        for r in range(t):                   # in two-shot every rank's x is assembled from slices that the other ranks computed
            assert same(xs[r][:T], ref), f"x of rank {r} vs the rank-ordered sum: {w}"
            assert (xs[r][T:].view(torch.int16) == BF16_NAN).all(), f"x past T x H of rank {r}: {w}"
        if two_shot:
            assert same(xs[0][:T], one), f"two-shot vs one-shot: {what}"
            # slice r: one contiguous run of gather[r], in rank order, together covering T x H exactly once; nothing else written
            start = 0
            for r in range(t):
                g = gath[r].view(torch.int16).flatten()
                wr = g != BF16_NAN
                n = int(wr.sum())
                if n:
                    lo = int(wr.int().argmax())
                    assert lo == start and bool(wr[lo:lo + n].all()), f"slice of rank {r} is not one run at {start}: {w}"
                    assert same(gath[r].flatten()[lo:lo + n], ref.flatten()[lo:lo + n]), f"gather of rank {r}: {w}"
                start += n
            assert start == T * H, f"the slices cover {start} of {T * H} elements: {w}"
        else:
            one = xs[0][:T].clone()
        del xs, gath


@pytest.mark.parametrize("case", CASES)
def test_prefill_all_reduce(L, case):
    H, t = CASES[case][0], CASES[case][6]
    for T in PREFILL_T:
        check_prefill(L, t, T, H, seed_of(case, T), f"{case} T {T}", must_reorder=True)
        torch.cuda.empty_cache()


@pytest.mark.parametrize("t,T,H", SYNTHETIC)
def test_prefill_all_reduce_short_slices(L, t, T, H):
    check_prefill(L, t, T, H, seed_of(t, T, H), f"t {t} T {T} H {H}", must_reorder=False)


# ------------------------------------------------------------------------------------------------ vocab-parallel greedy arg-max
ARGMAX_MS = [1, 12, 129, 256]


@pytest.mark.parametrize("case", ["qwen2.5-32b/tp4", "qwen2.5-32b/tp8", "llama-3-70b/tp8"])
def test_vocab_parallel_argmax(L, sms, case):
    H, _, _, _, _, V, t = CASES[case]
    K, Vs = H, V // t
    g = gen(seed_of(case, "lm"))
    B = (torch.randn(V, K, device=dev(), generator=g) * 0.1).to(BF16)
    rb = (t // 2) * Vs                       # a shard boundary
    j0, j1 = 37, (t - 1) * Vs + 101          # shard 0 and shard t-1
    B[rb] = B[rb - 1]; B[j1] = B[j0]        # exact ties across shards
    A = torch.randn(MAXM, K, device=dev(), generator=g).to(BF16)
    A[0] = A[5] = (B[rb - 1].float() * 10).to(BF16)      # rows whose largest logits are the ties
    A[6] = A[7] = (B[j0].float() * 10).to(BF16)
    words = (V + 31) // 32
    allowed = torch.zeros(7, words * 32, dtype=torch.bool, device=dev())
    allowed[0] = torch.rand(words * 32, device=dev(), generator=g) < 0.3    # a sparse grammar state
    allowed[1, V - 1] = True                  # only the last id
    allowed[2, Vs] = True                     # only the first id of shard 1
    # slot 3 allows nothing
    allowed[4, [rb - 1, rb]] = True           # a tie across a shard boundary
    allowed[5, [j0, j1]] = True               # a tie between shard 0 and shard t-1
    allowed[6, (t - 1) * Vs] = True           # only the first id of the last shard
    allowed[:, V:] = False
    table = torch.from_numpy(np.packbits(allowed.cpu().numpy(), axis=1, bitorder="little").view(np.int32).copy()).to(dev())
    slot = torch.tensor([-1, 0, 1, 2, 3, 4, 5, -1, -1, 6, 0, 3], dtype=torch.int32)
    slot = torch.cat([slot, torch.randint(-1, 7, (MAXM - len(slot),), generator=torch.Generator().manual_seed(t), dtype=torch.int32)]).to(dev())
    ref = torch.cat([A.double() @ B[r * Vs:(r + 1) * Vs].double().T for r in range(t)], 1)
    # the bound of test_masked_argmax (random signs), plus the accumulation bound of the sum of |products|: rows 0 and 5 .. 7 add K positive
    # products on their tied columns (the fp32 tensor-core accumulation truncates)
    tol = 1e-4 * K ** 0.5 + 1e-5 * ref.abs() + ACC_TOL_BF16_PER_K * K * torch.cat(
        [A.float().abs() @ B[r * Vs:(r + 1) * Vs].float().abs().T for r in range(t)], 1).double()
    allowed = allowed[:, :V]
    cols = torch.arange(V, device=dev())

    def first_max(lg, ok, n):
        """(max of lg over ok, lowest column reaching it; n when nothing is allowed)"""
        lg = torch.where(ok, lg, torch.tensor(-float("inf"), device=dev()))
        mx = lg.max(1, keepdim=True).values
        return mx[:, 0], torch.where(ok & (lg == mx), cols[None, :n], n).min(1).values

    for M in ARGMAX_MS:
        for bn in ((0, 64, 128, 256) if M == 12 else (0,)):
            for masked in ((True, False) if M == 12 else (True,)):
                what = f"{case} M {M} bn {bn} {'masked' if masked else 'no mask'}"
                logits = torch.full((M, V), float("nan"), dtype=torch.float32, device=dev())
                pairs = [torch.full((M, 2), -7, dtype=torch.int32, device=dev()) for _ in range(t)]
                ids = torch.full((M,), -1, dtype=torch.int32, device=dev())
                rc = L.oa_k_tp_lm_head_argmax(t, ptr(A), ptr(B), M, V, K, bn, ptr(table) if masked else None, ptr(slot) if masked else None,
                                              words, ptr(logits), parr(pairs), ptr(ids), None)
                assert rc == 0, (what, rc, _lib.last_error())
                assert ((logits.double() - ref[:M]).abs() <= tol[:M]).all(), f"logits: {what}"
                assert torch.equal(logits[:, rb - 1], logits[:, rb]) and torch.equal(logits[:, j0], logits[:, j1]), f"tied logits: {what}"
                ok = torch.ones(M, V, dtype=torch.bool, device=dev())
                if masked:
                    sl = slot[:M]
                    ok[sl >= 0] = allowed[sl[sl >= 0].long()]
                for r in range(t):                # each shard's pair: (max allowed logit, lowest global id), (-inf, r V/t) when none
                    s = slice(r * Vs, (r + 1) * Vs)
                    mx, first = first_max(logits[:, s], ok[:, s], Vs)
                    none = first == Vs
                    exp_v = torch.where(none, torch.tensor(-float("inf"), device=dev()), mx)
                    exp_i = torch.where(none, 0, first) + r * Vs
                    assert torch.equal(pairs[r][:, 0].view(torch.float32), exp_v), f"pair values of shard {r}: {what}"
                    assert torch.equal(pairs[r][:, 1].long(), exp_i), f"pair ids of shard {r}: {what}"
                _, first = first_max(logits, ok, V)
                exp = torch.where(first == V, 0, first)
                assert torch.equal(ids.long(), exp), f"ids: {what}: {ids.tolist()[:16]} vs {exp.tolist()[:16]}"
                assert ids[0].item() == rb - 1, f"a tie across the shard boundary takes the lower id: {what}"
                if M >= 12 and masked:
                    assert ids[2].item() == V - 1 and ids[3].item() == Vs and ids[4].item() == 0 and ids[9].item() == (t - 1) * Vs, what
                    assert ids[5].item() == rb - 1 and ids[6].item() == j0 and ids[7].item() == j0, f"ties across shards: {what}"
                    assert all(pairs[r][4, 0].view(torch.float32).item() == -float("inf") and pairs[r][4, 1].item() == r * Vs for r in range(t))


# ------------------------------------------------------------------------------------------------ refusals
def test_tp_entry_points_refuse_bad_shapes(L, sms):
    """t outside 2..8, a row length (H, K) that is not a multiple of 8, V % t, (V / t) % 8 and a launcher's refusal return a bad request
    before anything runs: no output changes"""
    BAD = _lib.OA_ERR_BAD_REQUEST
    n = 9
    A = [torch.randn(MAXM, 64, device=dev()).to(BF16) for _ in range(n)]
    B = [torch.randn(64, 64, device=dev()).to(BF16) for _ in range(n)]
    gain = torch.ones(64, dtype=BF16, device=dev())

    def rp(t, M=5, H=64, bn=128):
        parts = [torch.zeros(MAXM, 64, device=dev()) for _ in range(n)]
        xs = [torch.ones(MAXM, 64, dtype=BF16, device=dev()) for _ in range(n)]
        xns = [torch.zeros(MAXM, 64, dtype=BF16, device=dev()) for _ in range(n)]
        flags = new_flags()
        rc = L.oa_k_tp_row_parallel(t, parr(A), parr(B), M, H, 64, bn, sms, 0, parr(parts), parr(xs), parr(xns), ptr(gain), EPS, ptr(flags), 1, 1, None)
        assert all(not p.any() for p in parts) and all((x == 1).all() for x in xs) and all(not x.any() for x in xns), (t, M, H, bn)
        assert (flags == FLAG_FILL).all(), (t, M, H, bn)
        return rc

    def pf(t, H=64, two_shot=1):
        parts = [torch.ones(4, 64, dtype=BF16, device=dev()) for _ in range(n)]
        xs = [torch.zeros(4, 64, dtype=BF16, device=dev()) for _ in range(n)]
        gath = [torch.zeros(4, 64, dtype=BF16, device=dev()) for _ in range(n)]
        rc = L.oa_k_tp_allreduce_prefill(t, parr(parts), parr(xs), parr(gath), 4, H, two_shot, None)
        assert all(not x.any() for x in xs + gath), (t, H)
        return rc

    def lm(t, V, K=64):
        Bv = torch.randn(max(V, 8), 64, device=dev()).to(BF16)
        logits = torch.zeros(5, max(V, 8), device=dev())
        pairs = [torch.zeros(5, 2, dtype=torch.int32, device=dev()) for _ in range(n)]
        ids = torch.full((5,), -1, dtype=torch.int32, device=dev())
        rc = L.oa_k_tp_lm_head_argmax(t, ptr(A[0]), ptr(Bv), 5, V, K, 0, None, None, 0, ptr(logits), parr(pairs), ptr(ids), None)
        assert not logits.any() and all(not p.any() for p in pairs) and (ids == -1).all(), (t, V, K)
        return rc

    for t in (-1, 0, 1, 9):
        assert rp(t) == BAD and pf(t) == BAD and pf(t, two_shot=0) == BAD and lm(t, 64) == BAD, t
    assert rp(2, H=60) == BAD and pf(2, H=60) == BAD and lm(2, 64, K=60) == BAD
    assert lm(3, 64) == BAD and lm(4, 48) == BAD                 # V % t, (V / t) % 8
    assert rp(2, M=129, bn=256) == BAD                          # two 128-row slots take block_n 128 only
