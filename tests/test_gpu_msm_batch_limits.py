"""GPU: the branches of b200_msm_device_batch that exist because of device limits and large shapes, each reached on the
device and checked against known discrete logs.  The bases tile a pool of 256 minted points k_j*G, so record p must be
(sum_i s_(p,i) k_(i mod 256))*G: one CPU scalar multiplication per distinct vector, no GPU output in an expectation.
  - tail launches split into chunks of at most 65535 (vector, group) rows (for_each_tail_chunk), each with its own
    pointer offsets and y mod G: the rows / columns / planes tail (c >= 7) and the batched segment tail (c < 7);
  - the batched segment tail below c = 7 with 1, 2 or all window rows stored;
  - the multi-block counter scan whose chunk doubles beyond 1024 blocks (more than 2^26 counters);
  - window sizes 19-24, which the automatic choice never makes;
  - scratch regrowth while the set's previous batch is still queued, and at exactly the batch's size when the union of
    the old and the new shape would reach 2^31 sort entries, with b200_msm_device calls in between;
  - the staged backward pass under batches, prefixes n = 0 and n = 1, and skewed vectors next to uniform ones.
Each branch test shows by the launch counter that it ran: against a k = 2 batch of the same set, a batch of k vectors
issues launches(2) + ([m_k > 64 Ki] - [m_2 > 64 Ki]) + (chunks_k - 1) * (2 if c >= 7 else 1) launches, with
m_k = k*G*2^(c-1) + 1 counters (G window groups per vector).  The shape rules are restated here and checked without a
GPU: every case crosses the boundary it is named for."""
import functools

import numpy as np
import pytest

import test_gpu_msm_adversarial as adv
import test_gpu_msm_batch as tb
from oracle import ref_py as o
from test_gpu_msm_batch import L, pools  # noqa: F401  (fixtures: the library, the minted pools)

R = o.R
POOL = tb.POOL
gpu = pytest.mark.gpu

# ---- the library's batch rules, restated (capi.cu / msm.cuh) --------------------------------------------------------
MAX_ROWS = 65535          # kMaxGridY: (vector, group) rows per launch of a tail kernel
SCAN_CHUNK = 1 << 16      # msm_sort: counters one scan block walks before the chunk doubles
SCAN_BLOCKS = 1024        # kScanBlocks: at most this many scan blocks
ENTRY_LIMIT = 1 << 31     # batch_fits: sort entries (and buckets) of a batch scratch


def tail_chunks(k, G, max_rows=MAX_ROWS):
    """for_each_tail_chunk: [(y0, rows)] launches over the k*G (vector, group) rows, each a multiple of G rows."""
    rows, whole = k * G, max_rows // G
    chunk = max(whole, 1) * G
    return [(y0, min(chunk, rows - y0)) for y0 in range(0, rows, chunk)]


def counters(k, G, c):
    """Counters the sort of a batch scans: bucket 0 and k*G*2^(c-1) buckets."""
    return k * G * (1 << (c - 1)) + 1


def scan_split(m):
    """msm_sort: (chunk, blocks) of the counter scan of a batch; one block up to 64 Ki counters."""
    if m <= SCAN_CHUNK:
        return m, 1
    chunk = SCAN_CHUNK
    while -(-m // chunk) > SCAN_BLOCKS:
        chunk *= 2
    return chunk, -(-m // chunk)


def extra_launches(k, G, c):
    """launches(k) - launches(2) of batches on one set."""
    multi = lambda kk: int(counters(kk, G, c) > SCAN_CHUNK)
    return multi(k) - multi(2) + (len(tail_chunks(k, G)) - 1) * (2 if c >= 7 else 1)


def batch_fits(k, n, c, G):
    return k * adv.n_windows(c) * n < ENTRY_LIMIT and k * G * (1 << (c - 1)) + 3 < ENTRY_LIMIT


def regrown(cap, k, n, c, G):
    """batch_scratch: the (vectors, terms) capacity of a set's batch scratch after a batch of k vectors of n terms, from
    the capacity `cap` before it (None: no batch yet).  It grows to the larger of both in each dimension, or to exactly
    this batch's size when that union does not fit."""
    n = max(n, 1)
    if cap and cap[0] >= k and cap[1] >= n:
        return cap
    if cap and batch_fits(max(k, cap[0]), max(n, cap[1]), c, G):
        return max(k, cap[0]), max(n, cap[1])
    return k, n


def xyzz_batch_bytes(g, cap, c, G):
    """Device bytes of the batch scratch of an XYZZ set with capacity cap = (vectors, terms): sort_alloc, bucket_alloc
    and the scan totals."""
    k, n = cap
    rec = 4 * 32 * g                                            # XYZZ<Fq> / XYZZ<Fq2>
    nb = 1 << (c - 1)
    B = k * G * nb
    entries = k * adv.n_windows(c) * n
    slices = B + B // 2 + 2
    sort = 4 * ((B + 2) + (B + 3) + (B + 2) + entries + (B + 3) + 2 * slices)
    nseg = nb // (4 if nb >= 256 else 1)
    bits = c - 1
    kl = (bits + 1) // 2
    tail = k * G * ((1 << (bits - kl)) + (1 << kl) + bits + 1)
    return sort + rec * (B + slices + max(k * G * nseg + 1024, tail)) + 8 * SCAN_BLOCKS


def xyzz_set_bytes(g, n, c):
    """Device bytes of an XYZZ set with full tables before its first batch (bases_create)."""
    fe = 32 * g
    nwin, nb = adv.n_windows(c), 1 << (c - 1)
    slices = nb + nb // 2 + 2
    sort = 4 * ((nb + 2) + (nb + 3) + (nb + 2) + nwin * n + (nb + 3) + 2 * slices)
    nseg = nb // (4 if nb >= 256 else 1)
    bits = c - 1
    kl = (bits + 1) // 2
    tail = (1 << (bits - kl)) + (1 << kl) + bits + 1
    return nwin * n * 2 * fe + n * 32 + sort + 4 * fe * (nb + slices + max(nseg + 1024, tail)) + 4 * fe + 3 * fe + 4


# ---- vectors, launches and records ----------------------------------------------------------------------------------
def family(n, c, count, seed):
    """`count` distinct (n, 4) scalar vectors, every value < r: the digit extremes of window size c, all r - 1, then
    full width with 0, 1 and r - 1 mixed in (vectors of at least 3 terms)."""
    from gosnark_b200._lib import ints_to_limbs
    rng = np.random.default_rng(seed)
    out = [np.ascontiguousarray(adv.const(n, R - 1))]
    if n >= 6:
        out.insert(0, adv.scalar_families(n, c, seed)["digits"])
    while len(out) < count:
        v = adv.full_width(n, rng)
        if n >= 3:
            v[rng.choice(n, 3, replace=False)] = ints_to_limbs([0, 1, R - 1])
        out.append(v)
    return np.stack(out[:count])


def pick(k, count, seed):
    """Family index of each of k vectors: random, and no two neighbours equal, so a chunk that starts a vector too early
    or too late gives a wrong record."""
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, count, k)
    for p in range(1, k):
        if idx[p] == idx[p - 1]:
            idx[p] = (idx[p - 1] + 1 + rng.integers(0, count - 1)) % count
    return idx


def dlog_of(ks, vec):
    """sum_i s_i k_(i mod 256) mod r of one (n, 4) vector: column sums for whole pools, Python integers for prefixes."""
    if vec.shape[0] % len(ks) == 0:
        return adv.dlog(ks, vec)
    from gosnark_b200._lib import limbs_to_ints
    return sum(s * ks[i % len(ks)] for i, s in enumerate(limbs_to_ints(vec))) % R


@functools.lru_cache(maxsize=None)
def expect(g, d):
    return adv.expect_affine(g, d)


def load(g, pts, n, c=0, mode=0, t=0):
    from gosnark_b200 import bn128
    tiled = np.ascontiguousarray(pts[np.arange(n) % pts.shape[0]])
    return bn128.BaseSet(g, limbs=tiled, window_bits=c, acc_mode=mode, table_windows=t)


def groups_of(bs):
    nwin = bs.info()["n_windows"]
    return -(-nwin // bs.table_windows())


def fetch(bs, d_out):
    return d_out.cpu().numpy().view(np.uint64).reshape(-1, adv.REC_WORDS[bs.group])


def run(bs, stack, n=None):
    """b200_msm_device_batch over the k vectors of `stack` (k, N, 4) laid N scalars apart, over the first n (default N)
    bases; the raw records (k, 16 or 32)."""
    import torch
    k, N = stack.shape[0], stack.shape[1]
    d_s = tb.to_dev(stack.reshape(-1, 4))
    d_out = torch.full((k * adv.REC_WORDS[bs.group],), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    bs.msm_device_batch(d_s, N if n is None else n, k, d_out, stride=N)
    torch.cuda.synchronize()
    return fetch(bs, d_out)


def counted(lib, fn):
    """(kernel launches the library counts for fn(), fn's value)."""
    got = []
    count = adv.launches_of(lib, lambda: got.append(fn()))
    return count, got[0]


def check(g, recs, exps):
    """Every record decoded (words seen before are decoded once) and equal to its expected point."""
    assert len(recs) == len(exps)
    seen = {}
    for p, words in enumerate(recs):
        key = words.tobytes()
        if key not in seen:
            seen[key] = adv.decode_record(g, words)
        assert seen[key] == exps[p], p


def family_case(bs, ks, fam, k, seed):
    """(stack, expected points) of k vectors drawn from `fam`, one expectation per distinct vector."""
    exps = [expect(bs.group, dlog_of(ks, v)) for v in fam]
    assert len(set(exps)) == len(fam)
    idx = pick(k, len(fam), seed)
    return fam[idx], [exps[i] for i in idx]


# ---- shape rules, no GPU ---------------------------------------------------------------------------------------------
def test_cases_cross_the_boundaries_they_are_named_for():
    """Each (c, t, k) of the GPU cases below reaches the branch it is named for, by the restated rules."""
    # chunked rows / columns / planes tail, c = 7: t = 1 (G = 37, chunks of 1771 vectors) and full tables (G = 1)
    assert adv.n_windows(7) == 37
    assert tail_chunks(1771, 37) == [(0, 65527)]
    assert tail_chunks(1772, 37) == [(0, 65527), (65527, 37)]
    assert tail_chunks(3543, 37) == [(0, 65527), (65527, 65527), (131054, 37)]
    assert tail_chunks(65535, 1) == [(0, 65535)]
    assert tail_chunks(65536, 1) == [(0, 65535), (65535, 1)]
    assert [extra_launches(k, 37, 7) for k in (1771, 1772, 3543)] == [1, 3, 5]
    assert [extra_launches(k, 1, 7) for k in (65535, 65536)] == [1, 3]
    # chunked segment tail, c = 6, t = 1 (G = 43, chunks of 1524 vectors): one launch per further chunk
    assert adv.n_windows(6) == 43
    assert tail_chunks(1524, 43) == [(0, 65532)]
    assert tail_chunks(1525, 43) == [(0, 65532), (65532, 43)]
    assert [extra_launches(k, 43, 6) for k in (1524, 1525)] == [1, 2]
    # unchunked segment tails: c < 7, every t, k <= 16 stays in one chunk and one scan block
    for c in (4, 5, 6):
        nwin = adv.n_windows(c)
        for t in (1, 2, nwin):
            G = -(-nwin // t)
            assert all(extra_launches(k, G, c) == 0 for k in (2, 3, 16)), (c, t)
    # neighbouring vectors differ, so every chunk boundary has distinct vectors on both sides
    for k, seed in ((3543, 1), (65536, 2), (1525, 3)):
        idx = pick(k, 16, seed)
        assert np.all(idx[1:] != idx[:-1])
    # doubled scan chunk: c = 24 full tables, k = 8 needs 1025 blocks of 64 Ki, so the chunk doubles to 2^17 and the
    # last of 513 blocks holds one counter, bucket B*k: digit +2^23 of vector 7
    B = 1 << 23
    m = counters(8, 1, 24)
    assert m == (1 << 26) + 1 and -(-m // SCAN_CHUNK) == 1025
    chunk, blocks = scan_split(m)
    assert (chunk, blocks) == (1 << 17, 513) and m - (blocks - 1) * chunk == 1
    assert (7 * 1 + 0) * B + (1 << 23) == B * 8 == m - 1
    top = adv.digit_patterns(24)[0]
    assert adv.signed_digits(top, 24)[0][1] == 1 << 23
    assert scan_split(counters(4, 1, 24)) == (SCAN_CHUNK, 513)       # undoubled, its last block also one counter
    assert scan_split(counters(2, 1, 24))[1] > 1 and extra_launches(8, 1, 24) == 0
    # wide windows: the automatic choice stops at 18 for every set size
    assert max(adv.pick_window_bits(1 << e) for e in range(27)) <= 18
    assert all(adv.affine_slice_size(1 << 20, c) for c in (19, 20))   # forced batched affine still runs at 2^20
    # regrowth: at G1 2^20 (c = 17, 15 windows) 160 one-term vectors and one 2^20-term vector each fit, their union not
    c, N = adv.pick_window_bits(1 << 20), 1 << 20
    assert (c, adv.n_windows(c)) == (17, 15)
    assert batch_fits(160, 1, c, 1) and batch_fits(1, N, c, 1) and not batch_fits(160, N, c, 1)
    caps = []
    cap = None
    for k, n in REGROWTH:
        cap = regrown(cap, k, n, c, 1)
        caps.append(cap)
    assert caps == [(4, N), (9, N), (160, 1), (1, N), (160, 1), (2, N), (2, N)]
    # skew: the all-equal vector puts n entries in one bucket per window; both kernels cut it into more than kMergeSeq
    # slices
    for n in (1 << 20, 1 << 18):
        c = adv.pick_window_bits(n)
        assert n // adv.affine_slice_size(n, c) > adv.MERGE_SEQ and n // adv.xyzz_cap(n, c) > adv.MERGE_SEQ


# ---- 1. chunked rows / columns / planes tail (c >= 7) ----------------------------------------------------------------
@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("g", [1, 2])
def test_chunked_rowcol_planes_tail(L, pools, g):
    """c = 7 with one stored window row (G = 37 groups per vector): k = 1771, 1772 and 3543 vectors fill one, two and
    three tail chunks of at most 65535 rows; every record is its vector's point."""
    ks, pts = pools(g)
    n, c = POOL, 7
    bs = load(g, pts, n, c, t=1)
    try:
        assert bs.info()["window_bits"] == c and groups_of(bs) == 37
        fam = family(n, c, 16, seed=70 + g)
        base, recs = counted(L, lambda: run(bs, fam[:2]))
        check(g, recs, [expect(g, dlog_of(ks, v)) for v in fam[:2]])
        for k in (1771, 1772, 3543):
            stack, exps = family_case(bs, ks, fam, k, seed=k + g)
            count, recs = counted(L, lambda: run(bs, stack))
            assert count == base + extra_launches(k, 37, c), (k, count, base)
            check(g, recs, exps)
    finally:
        bs.free()


@gpu
@pytest.mark.timeout(600)
def test_chunked_tail_full_tables(L, pools):
    """Full tables at c = 7 (G = 1): k = 65535 vectors fill one chunk, k = 65536 leave one row for a second; four terms
    per vector."""
    ks, pts = pools(1)
    n, c = 4, 7
    bs = load(1, pts, n, c)
    try:
        assert bs.info()["window_bits"] == c and groups_of(bs) == 1
        fam = family(n, c, 16, seed=74)
        base, recs = counted(L, lambda: run(bs, fam[:2]))
        check(1, recs, [expect(1, dlog_of(ks, v)) for v in fam[:2]])
        for k in (65535, 65536):
            stack, exps = family_case(bs, ks, fam, k, seed=k)
            count, recs = counted(L, lambda: run(bs, stack))
            assert count == base + extra_launches(k, 1, c), (k, count, base)
            check(1, recs, exps)
    finally:
        bs.free()


# ---- 2. batched segment tail (c < 7) ----------------------------------------------------------------------------------
@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("c", [4, 5, 6])
@pytest.mark.parametrize("g", [1, 2])
def test_segment_tail_below_c7(L, pools, g, c, mode):
    """c in {4, 5, 6} with 1, 2 or all window rows stored, k in {2, 3, 16}, under both accumulation kernels (2^10 terms:
    a mean bucket of at least 16 entries, so forced batched affine runs): every record is its vector's point and the
    launches do not change with k."""
    ks, pts = pools(g)
    n = 1 << 10
    nwin = adv.n_windows(c)
    for t in (1, 2, nwin):
        bs = load(g, pts, n, c, mode, t)
        try:
            assert bs.info()["window_bits"] == c and bs.acc_mode() == mode and bs.table_windows() == t
            G = groups_of(bs)
            base = None
            for k in (2, 3, 16):
                vecs = tb.vectors(n, k, 1000 * c + 100 * t + 10 * k + g + mode)
                count, recs = counted(L, lambda: tb.run_batch(L, bs, vecs))
                tb.check_records(g, ks, vecs, recs)
                base = count if base is None else base
                assert count == base + extra_launches(k, G, c), (t, k, count, base)
        finally:
            bs.free()


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("g", [1, 2])
def test_chunked_segment_tail(L, pools, g):
    """c = 6 with one stored window row (G = 43): k = 1524 vectors fill one chunk of the batched segment reduction,
    k = 1525 start a second (one more launch each, not two: the segment tail, not the rows / columns / planes tail)."""
    ks, pts = pools(g)
    n, c = POOL, 6
    bs = load(g, pts, n, c, t=1)
    try:
        assert bs.info()["window_bits"] == c and groups_of(bs) == 43
        fam = family(n, c, 16, seed=60 + g)
        base, recs = counted(L, lambda: run(bs, fam[:2]))
        check(g, recs, [expect(g, dlog_of(ks, v)) for v in fam[:2]])
        for k in (1524, 1525):
            stack, exps = family_case(bs, ks, fam, k, seed=k + 10 * g)
            count, recs = counted(L, lambda: run(bs, stack))
            assert count == base + extra_launches(k, 43, c), (k, count, base)
            check(g, recs, exps)
    finally:
        bs.free()


# ---- 3. the doubled scan chunk ----------------------------------------------------------------------------------------
@gpu
@pytest.mark.timeout(600)
def test_scan_chunk_doubles_past_1024_blocks(L, pools):
    """c = 24 with full tables, 2^23 buckets per vector, 256 terms: k = 8 has 2^26 + 1 counters, so the scan chunk
    doubles to 2^17 and the last of 513 blocks holds one counter, bucket 8 * 2^23, which vector 7's digit +2^23 fills
    (k = 4: 513 blocks of 64 Ki, the last also one counter).  Needs about 29 GB of device memory; b200_bases_device_bytes
    counts exactly the restated scratch."""
    import torch
    from gosnark_b200._lib import limbs_to_ints
    g, n, c = 1, POOL, 24
    need = xyzz_set_bytes(g, n, c) + xyzz_batch_bytes(g, (8, n), c, 1)
    free, _ = torch.cuda.mem_get_info()
    if free < need + (2 << 30):
        pytest.skip(f"needs {(need >> 30) + 2} GiB of free device memory, {free >> 30} GiB free")
    ks, pts = pools(g)
    bs = load(g, pts, n, c)
    try:
        assert bs.info()["window_bits"] == c and bs.acc_mode() == 2
        b0 = bs.device_bytes()
        assert b0 == xyzz_set_bytes(g, n, c), (b0, xyzz_set_bytes(g, n, c))
        fam = family(n, c, 8, seed=24)
        top = fam[0]                                              # the digit-extreme vector: digit +2^23 in window 0
        assert any(adv.signed_digits(s, c)[0][1] == 1 << 23 for s in limbs_to_ints(top))
        base, recs = counted(L, lambda: run(bs, fam[1:3]))
        check(g, recs, [expect(g, dlog_of(ks, v)) for v in fam[1:3]])
        for k in (4, 8):
            stack = np.concatenate([fam[1:k], top[None]])          # the last vector fills bucket k * 2^23
            count, recs = counted(L, lambda: run(bs, stack))
            assert count == base + extra_launches(k, 1, c), (k, count, base)
            check(g, recs, [expect(g, dlog_of(ks, v)) for v in stack])
            assert bs.device_bytes() - b0 == xyzz_batch_bytes(g, (k, n), c, 1)
    finally:
        bs.free()


# ---- 4. window sizes 19-24 --------------------------------------------------------------------------------------------
def wide_window_case(lib, bs, ks, c, names):
    """Single MSMs of the digit-extreme families, then a k = 3 batch of them against a k = 2 batch."""
    g, n = bs.group, bs.n
    fam = adv.scalar_families(n, c, seed=c + 10 * g)
    for name in names:
        assert bs.msm(limbs=fam[name]) == adv.expect_out(g, adv.dlog(ks, fam[name])), (c, name)
    vecs = [fam[x] for x in names[:3]]
    base, recs = counted(lib, lambda: tb.run_batch(lib, bs, vecs[:2]))
    tb.check_records(g, ks, vecs[:2], recs)
    count, recs = counted(lib, lambda: tb.run_batch(lib, bs, vecs))
    assert count == base + extra_launches(3, 1, c), (c, count, base)
    tb.check_records(g, ks, vecs, recs)


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("g,logn", [(1, 16), (2, 14)])
def test_wide_windows(L, pools, g, logn):
    """c = 19 .. 24 (the ABI's range beyond the automatic choice): single MSMs and a k = 3 batch of the digit-extreme
    scalars (every digit +2^(c-1), every digit -(2^(c-1) - 1), a carry rippling through all-ones windows), powers of two
    and r - 1."""
    ks, pts = pools(g)
    n = 1 << logn
    for c in (19, 20, 21, 22, 23, 24):
        bs = load(g, pts, n, c)
        try:
            assert bs.info()["window_bits"] == c
            wide_window_case(L, bs, ks, c, ("digits", "pow2", "r-1"))
        finally:
            bs.free()


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("c", [19, 20])
def test_wide_windows_at_2_20(L, pools, c, mode):
    """G1 2^20 at c = 19 and 20 under both accumulation kernels (a mean bucket of 56 / 26 entries: forced batched affine
    runs), with all-equal and 99.9 % zero scalars next to the digit extremes."""
    ks, pts = pools(1)
    bs = load(1, pts, 1 << 20, c, mode)
    try:
        assert bs.info()["window_bits"] == c and bs.acc_mode() == mode
        wide_window_case(L, bs, ks, c, ("digits", "equal", "sparse", "pow2"))
    finally:
        bs.free()


# ---- 5. regrowth behind queued work -----------------------------------------------------------------------------------
REGROWTH = [(4, 1 << 20), (9, 1 << 20), (160, 1), (1, 1 << 20), (160, 1), (2, 1 << 20), (2, 1 << 20)]


@gpu
@pytest.mark.timeout(600)
def test_regrowth_behind_queued_work(L, pools):
    """G1 2^20, XYZZ (c = 17), every call on one torch side stream with no host synchronisation between them:
    k = 4 then k = 9 vectors of 2^20 terms (the second grows the scratch while the first may still run); 160 one-term
    vectors, whose union with the 2^20-term shape would pass 2^31 sort entries, so the scratch is reallocated at exactly
    that size, then one 2^20-term vector, then the 160 again; then b200_msm_device calls between batches.  Every record
    is right and b200_bases_device_bytes follows the regrowth rule after each call."""
    import torch
    from gosnark_b200._lib import check as ok
    g, N = 1, 1 << 20
    ks, pts = pools(g)
    bs = load(g, pts, N, 0, 2)
    side = torch.cuda.Stream()
    try:
        c = bs.info()["window_bits"]
        assert c == 17 and bs.acc_mode() == 2
        b0 = bs.device_bytes()
        big = family(N, c, 3, seed=5)
        tiny = family(1, c, 16, seed=6)

        def words(k):
            return torch.full((k * adv.REC_WORDS[g],), -1, dtype=torch.int64, device="cuda")
        # every input and output buffer first: nothing below synchronises the host until all calls are queued
        calls = []
        for step, (k, n) in enumerate(REGROWTH):
            stack, exps = family_case(bs, ks, big if n == N else tiny, k, seed=step)
            calls.append(("batch", tb.to_dev(stack.reshape(-1, 4)), words(k), k, n, exps))
        single = [("single", tb.to_dev(v), words(1), 1, N, [expect(g, dlog_of(ks, v))]) for v in big[:2]]
        calls = calls[:-1] + [single[0], calls[-1], single[1]]     # single MSMs around the last batch
        torch.cuda.synchronize()
        cap = None
        for kind, d_s, d_out, k, n, _ in calls:
            if kind == "single":
                ok(L.b200_msm_device(bs.handle, d_s.data_ptr(), n, 0, d_out.data_ptr(), side.cuda_stream))
            else:
                bs.msm_device_batch(d_s, n, k, d_out, stride=n, stream=side)
                cap = regrown(cap, k, n, c, 1)
            assert bs.device_bytes() - b0 == xyzz_batch_bytes(g, cap, c, 1), (k, n, cap)
        side.synchronize()
        for _, _, d_out, _, _, exps in calls:
            check(g, fetch(bs, d_out), exps)
    finally:
        side.synchronize()
        bs.free()


# ---- 6. the staged backward pass under batches ------------------------------------------------------------------------
@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("staging", [1, 2])
@pytest.mark.parametrize("g,logn", [(1, 14), (2, 11)])
def test_staged_backward_pass_in_batches(L, pools, g, logn, staging):
    """k = 3 batches on a forced batched-affine set under B200_CFG_TMA_STAGING 1 (every round staged) and 2 (rounds
    >= 2): the records are the vectors' points, and the batch runs log2(S) >= 2 affine rounds (three launches each more
    than the XYZZ set of the same points)."""
    from gosnark_b200 import _lib
    ks, pts = pools(g)
    n = 1 << logn
    c = adv.pick_window_bits(n)
    S = adv.affine_slice_size(n, c)
    assert S >= 4
    aff, xy = load(g, pts, n, 0, 1), load(g, pts, n, 0, 2)
    try:
        assert (aff.acc_mode(), xy.acc_mode()) == (1, 2)
        vecs = tb.vectors(n, 3, 40 + g + staging)
        _lib.check(L.b200_config(_lib.CFG_TMA_STAGING, staging))
        la, recs = counted(L, lambda: tb.run_batch(L, aff, vecs))
        tb.check_records(g, ks, vecs, recs)
        lx, _ = counted(L, lambda: tb.run_batch(L, xy, vecs))
        assert la - lx == 3 * (S.bit_length() - 1), (la, lx, S)
    finally:
        _lib.check(L.b200_config(_lib.CFG_TMA_STAGING, 0))
        aff.free()
        xy.free()


# ---- 7. prefixes, and skew next to uniform vectors --------------------------------------------------------------------
@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g", [1, 2])
def test_prefixes_of_zero_and_one_term(L, pools, g, mode):
    """A fresh set's first batch has n = 0 (scratch sized for one term): every record is infinity, with two launches
    fewer than n = 1 (no recode, no scatter).  n = 1 reuses that scratch and gives s_(p,0) * P_0; then the whole set."""
    ks, pts = pools(g)
    n = 1 << (12 if g == 1 else 10)
    bs = load(g, pts, n, 0, mode)
    try:
        assert bs.acc_mode() == mode
        vecs = np.stack(tb.vectors(n, 3, 30 + g + mode))
        b0 = bs.device_bytes()
        l0, recs = counted(L, lambda: run(bs, vecs, n=0))
        check(g, recs, [None] * 3)
        b1 = bs.device_bytes()
        assert b1 > b0
        l1, recs = counted(L, lambda: run(bs, vecs, n=1))
        check(g, recs, [expect(g, dlog_of(ks, v[:1])) for v in vecs])
        assert l0 == l1 - 2 and bs.device_bytes() == b1
        if mode == 2:
            assert b1 - b0 == xyzz_batch_bytes(g, (3, 1), bs.info()["window_bits"], 1)
        check(g, run(bs, vecs), [expect(g, dlog_of(ks, v)) for v in vecs])
    finally:
        bs.free()


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g,logn", [(1, 20), (2, 18)])
def test_skewed_next_to_uniform(L, pools, g, logn, mode):
    """k = 3 at G1 2^20 / G2 2^18: all-equal scalars (n entries in one bucket per window, cut into more than kMergeSeq
    slices), uniform scalars and 99.9 % zeros.  Replacing a skewed vector by uniform scalars leaves the other two records
    the same points."""
    ks, pts = pools(g)
    n = 1 << logn
    c = adv.pick_window_bits(n)
    bs = load(g, pts, n, 0, mode)
    try:
        assert bs.acc_mode() == mode and bs.info()["window_bits"] == c
        fam = adv.scalar_families(n, c, seed=logn + mode)
        rng = np.random.default_rng(logn + 10 * mode)
        vecs = np.stack([fam["equal"], adv.full_width(n, rng), fam["sparse"]])
        before = run(bs, vecs)
        check(g, before, [expect(g, dlog_of(ks, v)) for v in vecs])
        for q in (0, 2):
            changed = vecs.copy()
            changed[q] = adv.full_width(n, rng)
            after = run(bs, changed)
            for p in range(3):
                if p != q:
                    assert adv.decode_record(g, after[p]) == adv.decode_record(g, before[p]), (q, p)
            check(g, after[q:q + 1], [expect(g, dlog_of(ks, changed[q]))])
    finally:
        bs.free()
