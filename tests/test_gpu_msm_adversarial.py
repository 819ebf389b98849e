"""GPU: the MSM on inputs built to reach the branches that random bases and random scalars reach only by chance.

Bases (all k*G with a known k, minted by b200_g*_mul_batch_bcast as a small pool and tiled over the set):
  equal       every base the same point: equal points meet in every pair of the batched-affine tree (doublings) and
              every slice of a bucket has the same sum (the slice merge must double);
  pm-pairs    P_j, -P_j side by side: pairs cancel (P = -Q) and identical scalars on a pair give infinity;
  chain       k_{j+1} = 2^c k_j: table[w][j+1] == table[w+1][j], so equal points reach one bucket from different windows;
  half-inf    about half the bases (0,0,0), the rest one point: an operand at infinity next to a finite one.
Scalars: all equal, all 1, all r-1, boolean (90 % zero), powers of two, signed-digit extremes of the set's window size
(every digit +2^(c-1), every digit -(2^(c-1)-1), a carry rippling through all-ones windows), 99.9 % zero, and equal
scalars on neighbouring bases.  At benchmark sizes one bucket per window then holds every term of the set.

Every expected value is one CPU scalar multiplication by sum s_i k_i mod r, summed here per pool entry over the exact
column sums of the scalar limbs (no GPU output enters an expectation).  The window size, the batched-affine slice size
S and the XYZZ slice cap are restated here from bases_create / msm_sort; the window size and the accumulation mode are
asserted per set, and S is pinned by the launch count (three launches per batched-affine round)."""
import ctypes
import random

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu

Q, R = o.Q, o.R
OG = {1: o.BN.G1, 2: o.BN.G2}
FIELD = {1: o.BN.Fq1, 2: o.BN.Fq2}
CURVE_B = {1: 3, 2: o.BN.twist_coef_b}
REC_WORDS = {1: 16, 2: 32}             # u64 words of an XYZZ record
MONT = 1 << 256
MONT_INV_Q = pow(MONT, -1, Q)
MERGE_SEQ = 24                         # bucket_affine.cuh kMergeSeq: slices a thread merges on its own


@pytest.fixture(scope="module")
def lib():
    import torch
    from gosnark_b200 import _lib
    _lib.init()
    assert torch.cuda.is_available()
    return _lib.lib()


# ---- the library's shape rules, restated ----------------------------------------------------------------------------
def n_windows(c):
    return (255 + c - 1) // c


def pick_window_bits(n):
    """capi.cu pick_window_bits: the automatic window size."""
    best, best_cost = 8, None
    for c in range(8, 19):
        cost = n_windows(c) * n * 10.0 + 2.0 * (1 << (c - 1)) * 14.0 * 4.0
        if best_cost is None or cost < best_cost:
            best, best_cost = c, cost
    return best


def affine_slice_size(n, c):
    """capi.cu bases_create with the batched-affine accumulation forced: the slice size S, 0 when the set falls back to
    XYZZ (mean bucket population below 16)."""
    mean = n_windows(c) * n // (1 << (c - 1))
    if mean < 16:
        return 0
    s = 8
    while s < 128 and s * 2 * 6 <= mean:
        s *= 2
    return s


def xyzz_cap(n_terms, c):
    """capi.cu msm_sort: entries per slice of the XYZZ accumulation (twice the mean bucket, at least 32)."""
    nb = 1 << (c - 1)
    mean = (n_windows(c) * n_terms + nb - 1) // nb
    return max(2 * mean, 4 * 8)


def signed_digits(s, c):
    """msm.cuh for_each_digit: [(raw, digit)] per window; raw is the window's bits plus the incoming carry."""
    half, mask = 1 << (c - 1), (1 << c) - 1
    out, carry = [], 0
    for w in range(n_windows(c)):
        raw = ((s >> (w * c)) & mask) + carry
        neg = raw > half
        out.append((raw, raw - (1 << c) if neg else raw))
        carry = 1 if neg else 0
    assert sum(d << (w * c) for w, (_, d) in enumerate(out)) == s
    return out


def digit_patterns(c):
    """Scalars < r at the digit extremes of window size c, each built over as many windows W as fit below r (the top
    window cannot hold these digits), and checked against signed_digits:
      top     every digit +2^(c-1) (the highest bucket)
      neg     every digit -(2^(c-1) - 1) (the highest negated bucket), the carry-out +1 in window W
      ripple  2^(cW) - 1: digit -1, then windows whose raw value is exactly 2^c (digit 0, carry 1), then +1 in window W
    and each again over W - 1 windows, so the carry-out lands in a different window."""
    half, nwin = 1 << (c - 1), n_windows(c)

    def fit(build):
        w = nwin
        while build(w) >= R:
            w -= 1
        return w

    top = lambda w: sum(half << (c * i) for i in range(w))
    neg = lambda w: (half + 1) + sum(half << (c * i) for i in range(1, w))
    ripple = lambda w: (1 << (c * w)) - 1
    out = []
    for name, build in (("top", top), ("neg", neg), ("ripple", ripple)):
        w_max = fit(build)
        assert w_max >= 2
        for w in (w_max, w_max - 1):
            s = build(w)
            d = signed_digits(s, c)
            if name == "top":
                assert [x for _, x in d] == [half] * w + [0] * (nwin - w), (c, name, w)
            elif name == "neg":
                assert [x for _, x in d] == [1 - half] * w + [1] + [0] * (nwin - w - 1), (c, name, w)
            else:
                assert [x for _, x in d] == [-1] + [0] * (w - 1) + [1] + [0] * (nwin - w - 1), (c, name, w)
                assert all(raw == 1 << c for raw, _ in d[1:w]), (c, name, w)
            out.append(s)
    return out


# ---- bases ----------------------------------------------------------------------------------------------------------
BASE_KINDS = ("equal", "pm-pairs", "chain", "half-inf")


def mint(g, ks):
    """Standard-form Jacobian limbs of k*G for each k (k = 0: the all-zero point at infinity)."""
    from gosnark_b200._lib import ints_to_limbs
    from gosnark_b200.synthetic import mint_points
    pts = mint_points(g, ints_to_limbs([k % R for k in ks]))
    pts[[i for i, k in enumerate(ks) if k % R == 0]] = 0
    return pts


def base_pool(g, kind, c, seed):
    """(dlogs, points) of a pool that is tiled over the set: base i is pool entry i % len(pool)."""
    rng = random.Random(seed)
    k = rng.randrange(1, R)
    if kind == "equal":
        ks = [k]
    elif kind == "pm-pairs":
        ks = []
        for _ in range(128):
            kj = rng.randrange(1, R)
            ks += [kj, R - kj]
    elif kind == "chain":
        ks = [k]
        for _ in range(255):
            ks.append(ks[-1] * (1 << c) % R)
    else:
        ks = [k if rng.random() < 0.5 else 0 for _ in range(64)]
        ks[0], ks[1] = k, 0
    return ks, mint(g, ks)


def load_tiled(g, pool_pts, n, mode, window_bits=0):
    from gosnark_b200 import bn128
    pts = np.ascontiguousarray(pool_pts[np.arange(n) % pool_pts.shape[0]])
    return bn128.BaseSet(g, limbs=pts, window_bits=window_bits, acc_mode=mode)


def dlog(pool_ks, limbs):
    """sum_i s_i k_(i mod P) mod r for scalar limbs (n, 4), n a multiple of P: exact column sums of 32-bit halves."""
    P = len(pool_ks)
    n = limbs.shape[0]
    assert n % P == 0
    halves = np.ascontiguousarray(limbs, dtype=np.uint64).view(np.uint32).reshape(n // P, P, 8)
    cols = halves.astype(np.uint64).sum(axis=0)                       # each < 2^32 * n <= 2^54: exact
    return sum(k * sum(int(cols[p, j]) << (32 * j) for j in range(8)) for p, k in enumerate(pool_ks)) % R


def expect_out(g, k):
    """b200_g*_msm's output for (k mod r)*G: (x, y, 1), the point at infinity all zero."""
    G = OG[g]
    k %= R
    if k == 0:
        return (0, 0, 0) if g == 1 else ((0, 0), (0, 0), (0, 0))
    a = G.affine(G.mul_scalar(G.G, k))
    return (a[0], a[1], 1) if g == 1 else (a[0], a[1], (1, 0))


# ---- scalars --------------------------------------------------------------------------------------------------------
def full_width(count, rng):
    """count scalars uniform below 2^253 (< r) as (count, 4) limbs."""
    a = rng.integers(0, 1 << 64, size=(count, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 61) - 1)
    return a


def const(n, v):
    from gosnark_b200._lib import ints_to_limbs
    return np.ascontiguousarray(np.tile(ints_to_limbs([v]), (n, 1)))


def scalar_families(n, c, seed):
    """name -> (n, 4) scalar limbs, every value < r."""
    from gosnark_b200._lib import ints_to_limbs
    rng = np.random.default_rng(seed)
    fam = {"equal": np.ascontiguousarray(np.tile(full_width(1, rng), (n, 1))), "ones": const(n, 1),
           "r-1": const(n, R - 1)}
    b = np.zeros((n, 4), np.uint64)
    b[:, 0] = rng.random(n) < 0.1
    fam["bool"] = b
    e = np.arange(n) % 254
    p2 = np.zeros((n, 4), np.uint64)
    p2[np.arange(n), e // 64] = np.left_shift(np.uint64(1), (e % 64).astype(np.uint64))
    fam["pow2"] = p2
    pats = ints_to_limbs(digit_patterns(c))
    fam["digits"] = np.ascontiguousarray(pats[np.arange(n) % pats.shape[0]])
    sp = np.zeros((n, 4), np.uint64)
    where = rng.choice(n, size=max(n // 1000, 1), replace=False)
    sp[where] = full_width(where.size, rng)
    fam["sparse"] = sp
    fam["pairs"] = np.ascontiguousarray(np.repeat(full_width(n // 2, rng), 2, axis=0))
    return fam


def nudge(limbs, i):
    """A copy with scalar i one larger (its low limb is below 2^64 - 1: no carry)."""
    out = limbs.copy()
    assert out[i, 0] != np.uint64((1 << 64) - 1)
    out[i, 0] += np.uint64(1)
    return out


# ---- structured bases x skewed scalars at benchmark sizes ------------------------------------------------------------
SHAPES = [(1, 14), (1, 20), (2, 11), (2, 18)]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", BASE_KINDS)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g,logn", SHAPES, ids=[f"G{g}-n{1 << lg}" for g, lg in SHAPES])
def test_structured_bases_and_skewed_scalars(lib, g, logn, mode, kind):
    """Every scalar family on the structured base set of 2^logn terms, under the batched-affine (1) and the XYZZ (2)
    accumulation at the automatic window size: the exact known-discrete-log point.  Identical scalars on the ± pairs
    give infinity, and moving one of them by 1 gives exactly ±k*G.  Linearity on a skewed pair: msm(s) + msm(s') equals
    msm(s + s')."""
    n = 1 << logn
    c = pick_window_bits(n)
    ks, pool = base_pool(g, kind, c, seed=1000 * g + logn + 7 * BASE_KINDS.index(kind))
    bs = load_tiled(g, pool, n, mode)
    try:
        assert bs.acc_mode() == mode
        assert bs.info()["window_bits"] == c
        fam = scalar_families(n, c, seed=logn + 10 * g)
        for name, s in fam.items():
            assert bs.msm(limbs=s) == expect_out(g, dlog(ks, s)), name
        moved = nudge(fam["pairs"], 5)
        if kind == "pm-pairs":
            assert dlog(ks, fam["pairs"]) == 0 and dlog(ks, moved) == ks[5]          # ks[5] = r - ks[4]: -P_4
        assert bs.msm(limbs=moved) == expect_out(g, dlog(ks, moved))
        # linearity: boolean + powers of two stays below 2^253 + 1 < r, limb by limb without a carry
        s1, s2 = fam["bool"], fam["pow2"]
        o1, o2, o12 = bs.msm(limbs=s1), bs.msm(limbs=s2), bs.msm(limbs=s1 + s2)
        d1, d2 = dlog(ks, s1), dlog(ks, s2)
        assert o12 == expect_out(g, d1 + d2)
        if d1 and d2 and (d1 - d2) % R and (d1 + d2) % R:      # two distinct finite points, not negatives: a chord
            G = OG[g]
            assert tuple(G.affine(G.add(o1, o2))[:2]) == tuple(o12[:2])
    finally:
        bs.free()


def test_dlog_column_sums_match_plain_sums(lib):
    """The column-sum expectation equals the plain sum_i s_i k_i over Python ints for every family and pool kind."""
    from gosnark_b200._lib import limbs_to_ints
    n, c = 1 << 10, 10
    for kind in BASE_KINDS:
        ks, _ = base_pool(1, kind, c, seed=3)
        for name, s in scalar_families(n, c, seed=4).items():
            plain = sum(a * ks[i % len(ks)] for i, a in enumerate(limbs_to_ints(s))) % R
            assert dlog(ks, s) == plain, (kind, name)


# ---- window sizes the tests did not run, at their digit extremes -----------------------------------------------------
SWEEP_C = [2, 3, 7, 8, 12, 15, 16, 17, 18]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("c", SWEEP_C)
@pytest.mark.parametrize("g,n", [(1, 1 << 12), (2, 1 << 10)], ids=["G1-n4096", "G2-n1024"])
def test_window_sweep_digit_extremes(lib, g, n, c, mode):
    """Explicit window sizes over the doubling-chain bases of that size: powers of two (one digit per scalar, in every
    window in turn) and the digit-extreme patterns (highest bucket, highest negated bucket, a carry rippling through
    all-ones windows into the window above).  A forced batched-affine set whose mean bucket holds fewer than 16 entries
    runs XYZZ; that choice is asserted."""
    ks, pool = base_pool(g, "chain", c, seed=50 + c + g)
    bs = load_tiled(g, pool, n, mode, window_bits=c)
    try:
        assert bs.info()["window_bits"] == c
        assert bs.acc_mode() == (1 if mode == 1 and affine_slice_size(n, c) else 2)
        fam = scalar_families(n, c, seed=c)
        for name in ("pow2", "digits", "ones", "r-1"):
            s = fam[name]
            assert bs.msm(limbs=s) == expect_out(g, dlog(ks, s)), name
        # each digit pattern alone on every term: the same digit sequence in every column of the bucket set
        for v in digit_patterns(c)[::2]:
            s = const(n, v)
            assert bs.msm(limbs=s) == expect_out(g, dlog(ks, s)), hex(v)
    finally:
        bs.free()


# ---- slice-merge boundaries ------------------------------------------------------------------------------------------
MERGE_SHAPE = {1: (1 << 14, 13), 2: (1 << 11, 10)}      # (terms, window bits)


def launches_of(L, fn):
    """Kernel launches the library counts for fn() (b200_profile)."""
    from gosnark_b200._lib import check
    out = (ctypes.c_double * 8)()
    check(L.b200_profile(1))
    try:
        check(L.b200_profile_read(out))       # reset the counters
        fn()
        check(L.b200_profile_read(out))
    finally:
        check(L.b200_profile(0))
    return int(out[6])


def first_ones(n, cnt):
    s = np.zeros((n, 4), np.uint64)
    s[:cnt, 0] = 1
    return s


@pytest.mark.timeout(600)
@pytest.mark.parametrize("g", [1, 2])
def test_slice_merge_boundaries_equal_slices(lib, g):
    """One bucket of equal points (every base the same P, scalar 1 on the first cnt terms, 0 elsewhere) cut into
    slices whose sums are equal, so the merge must double:
      batched affine  cnt = 24 S (24 slices: the last bucket a thread merges alone) and 24 S + 1 (25 slices: the warp
                      path), with S restated from bases_create and pinned by the launch count;
      XYZZ            cnt = cap (one slice), cap + 1 and 2 cap (two slices);
    and, in both, digit 1 in every window of every term: tens of thousands of entries, thousands of slices."""
    n, c = MERGE_SHAPE[g]
    ks, pool = base_pool(g, "equal", c, seed=77 + g)
    k = ks[0]
    aff = load_tiled(g, pool, n, 1, window_bits=c)
    xy = load_tiled(g, pool, n, 2, window_bits=c)
    try:
        assert (aff.acc_mode(), xy.acc_mode()) == (1, 2)
        S = affine_slice_size(n, c)
        assert S and 24 * S + 1 <= n
        probe = first_ones(n, n)
        la = launches_of(lib, lambda: aff.msm(limbs=probe))
        lx = launches_of(lib, lambda: xy.msm(limbs=probe))
        assert la - lx == 3 * (S.bit_length() - 1), (la, lx, S)     # three launches per round, log2(S) rounds
        cap = xyzz_cap(n, c)
        assert 2 * cap <= n
        every = sum(1 << (c * w) for w in range(n_windows(c) - 1))    # digit 1 in every window below the top
        assert [d for _, d in signed_digits(every, c)] == [1] * (n_windows(c) - 1) + [0]
        for bs, counts in ((aff, (n, MERGE_SEQ * S, MERGE_SEQ * S + 1)), (xy, (n, cap, cap + 1, 2 * cap))):
            for cnt in counts:
                assert bs.msm(limbs=first_ones(n, cnt)) == expect_out(g, cnt * k), (bs.acc_mode(), cnt)
            assert bs.msm(limbs=const(n, every)) == expect_out(g, n * every * k), bs.acc_mode()
    finally:
        aff.free()
        xy.free()


# ---- the device entry point ------------------------------------------------------------------------------------------
def decode_record(g, words):
    """XYZZ record (X, Y, ZZ, ZZZ; Montgomery form) -> affine (x, y), None for ZZ = 0.  Asserts ZZ^3 = ZZZ^2 and that a
    finite point is on the curve."""
    from gosnark_b200._lib import limbs_to_ints
    v = [x * MONT_INV_Q % Q for x in limbs_to_ints(np.asarray(words, dtype=np.uint64))]
    F = FIELD[g]
    X, Y, ZZ, ZZZ = v if g == 1 else [(v[2 * i], v[2 * i + 1]) for i in range(4)]
    if F.is_zero(ZZ):
        return None
    assert F.mul(F.square(ZZ), ZZ) == F.square(ZZZ), "ZZ^3 != ZZZ^2"
    x, y = F.mul(X, F.inverse(ZZ)), F.mul(Y, F.inverse(ZZZ))
    assert F.square(y) == F.add(F.mul(F.square(x), x), CURVE_B[g]), "not on the curve"
    return (x, y)


def expect_affine(g, k):
    k %= R
    return None if k == 0 else tuple(OG[g].affine(OG[g].mul_scalar(OG[g].G, k))[:2])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", [1, 2])
def test_device_entry_skewed_at_2_20(lib, mode):
    """b200_msm_device on a torch side stream, G1 at 2^20: all-equal scalars and 99.9 % zeros on equal bases, identical
    scalars on ± pairs (infinity) and the same with one scalar moved by 1."""
    import torch
    from gosnark_b200._lib import check
    g, n = 1, 1 << 20
    c = pick_window_bits(n)
    fam = scalar_families(n, c, seed=20)
    side = torch.cuda.Stream()
    d_out = torch.zeros(REC_WORDS[g], dtype=torch.int64, device="cuda")
    cases = {"equal": ("equal", "sparse"), "pm-pairs": ("pairs", "pairs+1")}
    for kind, names in cases.items():
        ks, pool = base_pool(g, kind, c, seed=2000 + mode)
        bs = load_tiled(g, pool, n, mode)
        try:
            assert bs.acc_mode() == mode
            for name in names:
                s = nudge(fam["pairs"], 5) if name == "pairs+1" else fam[name]
                d_s = torch.from_numpy(s.reshape(-1).view(np.int64)).cuda()
                d_out.fill_(-1)
                torch.cuda.synchronize()
                check(lib.b200_msm_device(bs.handle, d_s.data_ptr(), n, 0, d_out.data_ptr(), side.cuda_stream))
                side.synchronize()
                exp = dlog(ks, s)
                if name == "pairs":
                    assert exp == 0
                assert decode_record(g, d_out.cpu().numpy().view(np.uint64)) == expect_affine(g, exp), (kind, name)
        finally:
            bs.free()
