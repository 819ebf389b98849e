"""GPU: batches of MSMs over one base set (b200_msm_device_batch): k scalar vectors in one set of launches, record p the
MSM of vector p.  Every expected value comes from known discrete logs: the bases tile a pool of 256 minted points k_j*G,
so record p must be (sum_i s_(p,i) k_(i mod 256))*G, one CPU scalar multiplication (test_gpu_msm_adversarial's column
sums); no GPU output feeds an expectation.
  - G1 at 2^14 and 2^20, G2 at 2^11 and 2^18, k in {1, 3, 16}, under both accumulation kernels and t in {1, 3, all}
    stored window rows;
  - vectors with 0, 1 and r-1, all-zero vectors between non-zero ones, identical vectors, skewed (boolean) vectors, and
    Montgomery-form scalars;
  - changing vector q leaves every record p != q the same point, and k = 1 gives b200_msm_device's point (the counting
    sort orders the entries of a bucket by atomics, so the XYZZ representation of a sum may differ from run to run);
  - strides (0, n, larger than n), a torch side stream, the scratch growth counted by b200_bases_device_bytes, and the
    argument checks (k = 0, n beyond the set, the 2^31-entry capacity)."""
import numpy as np
import pytest

import test_gpu_msm_adversarial as adv
from oracle import ref_py as o

pytestmark = pytest.mark.gpu

R = o.R
EINVAL = -3
MONT = 1 << 256
POOL = 256


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


@pytest.fixture(scope="module")
def pools(L):
    made = {}

    def get(g):
        if g not in made:
            import random
            rng = random.Random(0xBA7 + g)
            ks = [rng.randrange(1, R) for _ in range(POOL)]
            made[g] = (ks, adv.mint(g, ks))
        return made[g]
    return get


def load(g, pool_pts, n, mode=0, t=0):
    from gosnark_b200 import bn128
    pts = np.ascontiguousarray(pool_pts[np.arange(n) % pool_pts.shape[0]])
    return bn128.BaseSet(g, limbs=pts, acc_mode=mode, table_windows=t)


def vectors(n, k, seed):
    """k (n, 4) scalar-limb vectors, every value < r: full width with 0 / 1 / r-1 mixed in, then an all-zero vector,
    a repeat of the first, full width again and boolean (skewed) ones, cycling."""
    rng = np.random.default_rng(seed)
    out = []
    for p in range(k):
        kind = p % 5
        if kind == 0 or kind == 3:
            v = adv.full_width(n, rng)
            v[rng.choice(n, 3, replace=False)] = np.stack([adv.const(1, 0)[0], adv.const(1, 1)[0], adv.const(1, R - 1)[0]])
        elif kind == 1:
            v = np.zeros((n, 4), np.uint64)
        elif kind == 2:
            v = out[0].copy()
        else:
            v = np.zeros((n, 4), np.uint64)
            v[:, 0] = rng.random(n) < 0.1
        out.append(np.ascontiguousarray(v))
    return out


def to_dev(arr):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def run_batch(L, bs, vecs, stride=None, mont=0, stream=None, n=None):
    """b200_msm_device_batch over the vectors laid `stride` scalars apart (the gap filled with values that must not be
    read); returns the raw record words, (k, 16 or 32)."""
    import torch
    k = len(vecs)
    n = vecs[0].shape[0] if n is None else n
    stride = n if stride is None else stride
    buf = np.full((max((k - 1) * stride + n, 1), 4), 0xFFFFFFFFFFFFFFFF, np.uint64)   # >= r: read as 0 if it were read
    for p, v in enumerate(vecs):
        buf[p * stride:p * stride + n] = v[:n]
    d_s = to_dev(buf)
    words = adv.REC_WORDS[bs.group]
    d_out = torch.full((k * words,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    bs.msm_device_batch(d_s, n, k, d_out, stride=stride, mont=mont, stream=stream)
    if stream is None:
        torch.cuda.synchronize()
    else:
        stream.synchronize()
    return d_out.cpu().numpy().view(np.uint64).reshape(k, words)


def check_records(g, ks, vecs, recs):
    for p, v in enumerate(vecs):
        assert adv.decode_record(g, recs[p]) == adv.expect_affine(g, adv.dlog(ks, v)), p


@pytest.mark.timeout(900)
@pytest.mark.parametrize("t", [1, 3, 0])
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g,logn", [(1, 14), (2, 11)])
def test_batch_known_discrete_logs(L, pools, g, logn, mode, t):
    """k in {1, 3, 16} at G1 2^14 / G2 2^11: every record is its vector's known-discrete-log point, under both
    accumulation kernels and with 1, 3 or all window rows stored; k = 1 gives b200_msm_device's point."""
    import torch
    ks, pts = pools(g)
    n = 1 << logn
    bs = load(g, pts, n, mode, t)
    try:
        for k in (1, 3, 16):
            vecs = vectors(n, k, 100 * k + 10 * g + mode + t)
            recs = run_batch(L, bs, vecs)
            check_records(g, ks, vecs, recs)
            if k == 1:
                d_rec = torch.zeros(adv.REC_WORDS[g], dtype=torch.int64, device="cuda")
                from gosnark_b200._lib import check
                d_s = to_dev(vecs[0])
                check(L.b200_msm_device(bs.handle, d_s.data_ptr(), n, 0, d_rec.data_ptr(), None))
                torch.cuda.synchronize()
                assert adv.decode_record(g, d_rec.cpu().numpy().view(np.uint64)) == adv.decode_record(g, recs[0])
    finally:
        bs.free()


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g,logn", [(1, 20), (2, 18)])
def test_batch_benchmark_sizes(L, pools, g, logn, mode):
    """G1 2^20 and G2 2^18 with all window rows, k in {1, 3, 16} under both accumulation kernels, and t = 3 with k = 3."""
    ks, pts = pools(g)
    n = 1 << logn
    bs = load(g, pts, n, mode)
    try:
        for k in (1, 3, 16):
            vecs = vectors(n, k, 7 * k + g + mode)
            check_records(g, ks, vecs, run_batch(L, bs, vecs))
    finally:
        bs.free()
    if mode == 2:
        bs = load(g, pts, n, mode, 3)
        try:
            vecs = vectors(n, 3, 99 + g)
            check_records(g, ks, vecs, run_batch(L, bs, vecs))
        finally:
            bs.free()


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g", [1, 2])
def test_changing_one_vector_leaves_the_other_records_unchanged(L, pools, g, mode):
    """Vector q replaced by other scalars: record q follows, every other record stays the same point (the vectors'
    buckets, slices and tails do not mix)."""
    ks, pts = pools(g)
    n = 1 << (13 if g == 1 else 11)
    bs = load(g, pts, n, mode)
    try:
        vecs = vectors(n, 6, 5 + g + mode)
        before = run_batch(L, bs, vecs)
        check_records(g, ks, vecs, before)
        for q in (0, 4):
            changed = list(vecs)
            changed[q] = adv.full_width(n, np.random.default_rng(q + 50))
            after = run_batch(L, bs, changed)
            for p in range(len(vecs)):
                if p != q:
                    assert adv.decode_record(g, after[p]) == adv.decode_record(g, before[p]), (q, p)
            assert adv.decode_record(g, after[q]) == adv.expect_affine(g, adv.dlog(ks, changed[q]))
    finally:
        bs.free()


@pytest.mark.parametrize("g", [1, 2])
def test_strides_prefix_montgomery_and_side_stream(L, pools, g):
    """stride > n with unread values between the vectors, stride 0 (every record the same MSM), a prefix n < the set's
    size, Montgomery-form scalars (s * 2^256 mod r), and a torch side stream."""
    import torch
    ks, pts = pools(g)
    n = 1 << (12 if g == 1 else 10)
    bs = load(g, pts, n)
    try:
        vecs = vectors(n, 4, 17 + g)
        check_records(g, ks, vecs, run_batch(L, bs, vecs, stride=n + 77))
        recs = run_batch(L, bs, [vecs[0]] * 5, stride=0)
        check_records(g, ks, [vecs[0]] * 5, recs)
        m = n // 2
        half = [v[:m] for v in vecs]
        check_records(g, ks, half, run_batch(L, bs, vecs, stride=n, n=m))
        from gosnark_b200._lib import ints_to_limbs, limbs_to_ints
        mont = [ints_to_limbs([s * MONT % R for s in limbs_to_ints(v)]) for v in vecs]
        check_records(g, ks, vecs, run_batch(L, bs, mont, mont=1))
        check_records(g, ks, vecs, run_batch(L, bs, vecs, stream=torch.cuda.Stream()))
    finally:
        bs.free()


@pytest.mark.parametrize("g", [1, 2])
def test_scratch_growth_and_argument_checks(L, pools, g):
    """The first batch allocates the batch scratch (b200_bases_device_bytes grows), a smaller batch reuses it, a larger
    one grows it.  k = 0, n beyond the set and k * nwin * n >= 2^31 sort entries return B200_EINVAL without allocating,
    and the set still computes afterwards."""
    import torch
    ks, pts = pools(g)
    n = 1 << 10
    bs = load(g, pts, n)
    try:
        b0 = bs.device_bytes()
        vecs = vectors(n, 4, 3 + g)
        check_records(g, ks, vecs, run_batch(L, bs, vecs))
        b1 = bs.device_bytes()
        assert b1 > b0
        check_records(g, ks, vecs[:2], run_batch(L, bs, vecs[:2]))
        assert bs.device_bytes() == b1
        more = vectors(n, 9, 4 + g)
        check_records(g, ks, more, run_batch(L, bs, more))
        b2 = bs.device_bytes()
        assert b2 > b1
        d_s = to_dev(vecs[0])
        d_out = torch.zeros(64 * adv.REC_WORDS[g], dtype=torch.int64, device="cuda")
        fn = L.b200_msm_device_batch
        assert fn(bs.handle, d_s.data_ptr(), n, 0, n, 0, d_out.data_ptr(), None) == EINVAL
        assert fn(bs.handle, d_s.data_ptr(), n + 1, 1, n, 0, d_out.data_ptr(), None) == EINVAL
        nwin = bs.info()["n_windows"]
        k_big = (1 << 31) // (nwin * n) + 1
        assert fn(bs.handle, d_s.data_ptr(), n, k_big, 0, 0, d_out.data_ptr(), None) == EINVAL
        assert fn(bs.handle, d_s.data_ptr(), n, 1, 1 << 32, 0, d_out.data_ptr(), None) == EINVAL
        assert fn(bs.handle, None, n, 1, n, 0, d_out.data_ptr(), None) == EINVAL
        assert bs.device_bytes() == b2
        check_records(g, ks, vecs, run_batch(L, bs, vecs))
    finally:
        bs.free()


@pytest.mark.parametrize("k", [64, 1024])
def test_launch_count_does_not_grow_with_k(L, pools, k):
    """A batch issues the kernel launches of one MSM (k = 1), plus one (k_scan_totals) once its k*2^(c-1) bucket counters
    exceed 64 Ki and the counter scan runs on several blocks (b200_profile_read's launch counter).  At n = 2^10 (c = 10)
    k = 64 stays below that and k = 1024 crosses it."""
    ks, pts = pools(1)
    n = 1 << 10
    bs = load(1, pts, n, 2)
    try:
        c = bs.info()["window_bits"]
        extra = 1 if k * (1 << (c - 1)) + 1 > 1 << 16 else 0
        assert extra == (k == 1024), c
        one = vectors(n, 1, 1)
        many = vectors(n, k, 2)
        counts = [adv.launches_of(L, lambda v=v: run_batch(L, bs, v)) for v in (one, many)]
        assert counts[1] == counts[0] + extra, counts
        check_records(1, ks, many[:5], run_batch(L, bs, many)[:5])
    finally:
        bs.free()
