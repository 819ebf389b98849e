"""CPU: batches of MSMs over one base set (b200_msm_device_batch) through every kernel on the CPU emulation
(tests/host/batch_msm_test.cpp, csrc/host_stub): the batched signed-digit recode and counting sort over k*G*2^(c-1)
buckets, the multi-block counter scan, both accumulation kernels, the slice merge and the per-vector tails.  Every record
is the oracle's sum_i s_(p,i) * P_i, for G1 and G2, k in {1, 2, 5}, t in {1, 2, nwin} and c below and above the c = 7
switch between the segment tail and the rows / columns / planes tail.  k = 1 through the batch sequence leaves the same
offsets, slice tables, sorted entries, buckets and record as the one-MSM sequence."""
import ctypes
import random

import numpy as np
import pytest

import build as b200build
from oracle import ref_py as o

R_ = o.R


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_batch_msm())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _flat(pts):
    flat = []
    for p in pts:
        for cc in p:
            flat.extend(cc if isinstance(cc, tuple) else (cc,))
    return flat


def _points(group, out, k):
    raw = out.tobytes()
    v = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(len(raw) // 32)]
    per = 3 if group == 1 else 6
    recs = [v[p * per:(p + 1) * per] for p in range(k)]
    return [(r[0], r[1], r[2]) if group == 1 else ((r[0], r[1]), (r[2], r[3]), (r[4], r[5])) for r in recs]


def _expect(group, k):
    G = o.BN.G1 if group == 1 else o.BN.G2
    if k % R_ == 0:
        return (0, 0, 0) if group == 1 else ((0, 0), (0, 0), (0, 0))
    e = G.affine(G.mul_scalar(G.G, k % R_))
    return (e[0], e[1], 1) if group == 1 else (e[0], e[1], (1, 0))


def _bases(group, n, seed):
    G = o.BN.G1 if group == 1 else o.BN.G2
    rng = random.Random(seed)
    ks = [rng.randrange(1, R_) for _ in range(n)]
    ks[3] = ks[4]                                           # a repeated point
    return ks, [G.mul_scalar(G.G, k) for k in ks]           # Jacobian, Z != 1


def _vectors(rng, n, k):
    """k scalar vectors: 0, 1 and r-1 mixed into random ones; with k >= 3 an all-zero vector between non-zero ones and
    two identical vectors; with k = 2 the second repeats the first."""
    def rand_vec():
        v = [rng.randrange(R_) for _ in range(n)]
        for i, s in zip(rng.sample(range(n), 3), (0, 1, R_ - 1)):
            v[i] = s
        return v
    if k == 1:
        return [rand_vec()]
    if k == 2:
        v = rand_vec()
        return [v, list(v)]
    vs = [rand_vec(), [0] * n, rand_vec()]
    vs.append(list(vs[2]))
    while len(vs) < k:
        vs.append([R_ - 1 if i % 2 else 1 for i in range(n)])
    return vs[:k]


def _run(lib, group, ks, pts, vecs, c, t, S, stride, scan_chunk, max_rows=65535):
    n, k = len(ks), len(vecs)
    rng = random.Random(n * k + stride)
    flat = []
    for p, v in enumerate(vecs):                            # the gap between vectors holds values that must not be read
        flat += v + ([rng.randrange(1, R_) for _ in range(stride - n)] if p + 1 < k else [])
    if stride == 0:
        flat = vecs[0]
    w = 8 if group == 1 else 16
    out = np.zeros(k * 3 * w, dtype=np.uint32)
    rc = lib.t_msm_batch(group, _ptr(_u32(_flat(pts))), _ptr(_u32(flat)), n, k, stride, c, t, S, scan_chunk, max_rows,
                         _ptr(out))
    assert rc == 0
    return _points(group, out, k)


CASES = [(1, 4, 0), (1, 5, 8), (1, 7, 0), (1, 8, 16), (2, 4, 0), (2, 5, 0), (2, 7, 0), (2, 8, 8)]


def _record_cases():
    """(group, c, S, t, k).  The segment tail (c < 7) runs the whole grid.  The rows / columns / planes tail emulates one
    CTA per (vector, window group) and costs ~30 s per vector at t = 1 on the CPU, so small t there is tested with fewer
    vectors."""
    small_t = {(1, 7, "1", 1), (1, 8, "2", 2)}
    out = []
    for group, c, S in CASES:
        for t in ("1", "2", "nwin"):
            for k in (1, 2, 5):
                full = t == "nwin" and not (group == 2 and c == 8 and k == 5)
                if c < 7 or full or (group, c, t, k) in small_t:
                    out.append((group, c, S, t, k))
    return out


@pytest.mark.parametrize("group,c,S,which_t,k", _record_cases())
def test_batch_records_equal_oracle(lib, group, c, S, which_t, k):
    """Record p is sum_i s_(p,i) * P_i for every vector; the vectors sit `stride` = n + 3 apart with unread values
    between them; batches of more than one vector scan their counters with several blocks of 300 counters."""
    nwin = (255 + c - 1) // c
    t = {"1": 1, "2": 2, "nwin": nwin}[which_t]
    n = 16 if group == 1 else 8
    ks, pts = _bases(group, n, 100 * group + 10 * c + t)
    vecs = _vectors(random.Random(1000 * k + 100 * group + c + t), n, k)
    got = _run(lib, group, ks, pts, vecs, c, t, S, n + 3, 300 if k > 1 else 0)
    for p, v in enumerate(vecs):
        assert got[p] == _expect(group, sum(a * s for a, s in zip(ks, v))), p


@pytest.mark.parametrize("group,c,S,t", [(1, 5, 0, 2), (1, 8, 16, 32), (2, 7, 0, 37)])
def test_stride_zero_reads_one_vector_k_times(lib, group, c, S, t):
    """stride = 0: every vector is the same n scalars, so all k records are that one MSM."""
    n = 16 if group == 1 else 8
    ks, pts = _bases(group, n, 7 + c)
    v = _vectors(random.Random(c), n, 1)[0]
    got = _run(lib, group, ks, pts, [v] * 4, c, t, S, 0, 300)
    exp = _expect(group, sum(a * s for a, s in zip(ks, v)))
    assert got == [exp] * 4


@pytest.mark.parametrize("group,c,S,t,max_rows", [(1, 4, 0, 2, 2 * 32 + 1), (1, 5, 8, 1, 51), (1, 7, 0, 37, 2),
                                                (1, 8, 16, 16, 3 * 2 + 1), (2, 5, 0, 51, 3)])
def test_tail_launches_split_into_row_chunks(lib, group, c, S, t, max_rows):
    """The (vector, window group) tail kernels split into launches of at most max_rows rows, each a whole number of
    vectors' groups (on the device: at most 65535, reached when k*G exceeds it).  Chunk boundaries inside the batch, with
    each chunk's own pointer offsets and y mod G scaling, give the same records as the oracle."""
    n = 16 if group == 1 else 8
    ks, pts = _bases(group, n, 11 * c + t)
    vecs = _vectors(random.Random(3 * c + t), n, 5)
    got = _run(lib, group, ks, pts, vecs, c, t, S, n, 300, max_rows)
    for p, v in enumerate(vecs):
        assert got[p] == _expect(group, sum(a * s for a, s in zip(ks, v))), p


@pytest.mark.parametrize("group,c,S,which_t", [(1, 4, 0, "1"), (1, 5, 8, "1"), (1, 7, 0, "nwin"), (1, 8, 16, "nwin"),
                                               (2, 5, 0, "1"), (2, 7, 0, "nwin")])
@pytest.mark.parametrize("scan_chunk", [0, 300])
def test_single_vector_batch_is_bit_identical(lib, group, c, S, which_t, scan_chunk):
    """k = 1 through the batch sequence, with one scan block or several, against the one-MSM sequence: the same
    offsets, slice tables, sorted entries and buckets byte for byte, and the same record (byte for byte where the tail
    launches are the same, c >= 7; the same point for c < 7, whose tree sum differs in shape)."""
    nwin = (255 + c - 1) // c
    t = 1 if which_t == "1" else nwin
    n = 24 if group == 1 else 12
    ks, pts = _bases(group, n, 5 * c + group)
    v = _vectors(random.Random(c + t), n, 1)[0]
    assert lib.t_batch_single_identical(group, _ptr(_u32(_flat(pts))), _ptr(_u32(v)), n, c, t, S, scan_chunk) == 0
