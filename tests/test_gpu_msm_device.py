"""GPU tests of the device-resident MSM entry points (include/b200snark.h):
  * b200_msm_device            scalars in device memory (standard or Montgomery form), the sum left on a stream as
                               an XYZZ record;
  * b200_g{1,2}_sum_partials   add `count` such records and normalise (what the multi-GPU path does after its
                               all-gather);
  * out-of-range inputs on the `_device` entry points: read as 0, reported by no later call.
Every point is P_i = k_i*G minted on the GPU, so every expected value is one CPU scalar multiplication by a known
discrete log (as in test_gpu_msm.py).  Records are decoded here, independently of the library: x = X/ZZ, y = Y/ZZZ
over Montgomery-form limbs, with ZZ^3 = ZZZ^2 and the curve equation checked for every finite point."""
import random

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu

Q, R = o.Q, o.R
OG = {1: o.BN.G1, 2: o.BN.G2}
FIELD = {1: o.BN.Fq1, 2: o.BN.Fq2}
CURVE_B = {1: 3, 2: o.BN.twist_coef_b}                # y^2 = x^3 + b (G2: the twist's b' = 3 / (9 + u))
WORDS = {1: 12, 2: 24}                               # u64 words of a standard-form Jacobian point
REC_WORDS = {1: 16, 2: 32}                           # u64 words of an XYZZ record: 128 B / 256 B
MONT = 1 << 256                                      # Montgomery radix of F_q and F_r
MONT_INV_Q = pow(MONT, -1, Q)
EINVAL = -3


@pytest.fixture(scope="module")
def lib():
    import torch
    from gosnark_b200 import _lib
    _lib.init()
    assert torch.cuda.is_available()
    return _lib.lib()


def to_dev(arr):
    """uint64 numpy array -> int64 CUDA tensor holding the same bytes (ready for use on any stream)."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def from_dev(t):
    return t.cpu().numpy().view(np.uint64)


def expect_affine(g, k):
    """Affine (x, y) of (k mod r)*G, None for the point at infinity."""
    k %= R
    if k == 0:
        return None
    return tuple(OG[g].affine(OG[g].mul_scalar(OG[g].G, k))[:2])


def expect_out(g, k):
    """The normalised output of sum_partials / b200_g*_msm for (k mod r)*G: (x, y, 1), infinity all-zero."""
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    a = expect_affine(g, k)
    if a is None:
        return _unflatten_g1(np.zeros(12, np.uint64))[0] if g == 1 else _unflatten_g2(np.zeros(24, np.uint64))[0]
    return (a[0], a[1], 1) if g == 1 else (a[0], a[1], (1, 0))


def unflatten(g, words):
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    return (_unflatten_g1 if g == 1 else _unflatten_g2)(words)


# ---- XYZZ records -------------------------------------------------------------------------------------------------
def decode_record(g, words):
    """Raw record words (X, Y, ZZ, ZZZ; little-endian limbs, Montgomery form; F_q^2 as (c0, c1)) -> affine (x, y),
    or None when ZZ = 0 (infinity).  Asserts ZZ^3 = ZZZ^2 and that a finite point is on the curve."""
    from gosnark_b200._lib import limbs_to_ints
    v = [c * MONT_INV_Q % Q for c in limbs_to_ints(np.asarray(words, dtype=np.uint64))]
    assert len(v) == (4 if g == 1 else 8)
    F = FIELD[g]
    X, Y, ZZ, ZZZ = v if g == 1 else [(v[2 * i], v[2 * i + 1]) for i in range(4)]
    if F.is_zero(ZZ):
        return None
    assert F.mul(F.square(ZZ), ZZ) == F.square(ZZZ), "ZZ^3 != ZZZ^2"
    x, y = F.mul(X, F.inverse(ZZ)), F.mul(Y, F.inverse(ZZZ))
    assert F.square(y) == F.add(F.mul(F.square(x), x), CURVE_B[g]), "not on the curve"
    return (x, y)


def encode_record(g, xy, z):
    """The record of affine point xy (None: all-zero infinity) under z: ZZ = z^2, ZZZ = z^3, X = x ZZ, Y = y ZZZ."""
    from gosnark_b200._lib import ints_to_limbs
    if xy is None:
        return np.zeros(REC_WORDS[g], np.uint64)
    F = FIELD[g]
    zz = F.square(z)
    zzz = F.mul(zz, z)
    coords = [F.mul(xy[0], zz), F.mul(xy[1], zzz), zz, zzz]
    flat = coords if g == 1 else [c for pair in coords for c in pair]
    return ints_to_limbs([c * MONT % Q for c in flat]).reshape(-1)


def rand_z(g, rng):
    return rng.randrange(2, Q) if g == 1 else (rng.randrange(Q), rng.randrange(1, Q))


def neg_affine(g, xy):
    return (xy[0], FIELD[g].neg(xy[1]))


# ---- base sets ----------------------------------------------------------------------------------------------------
def mint(g, n, seed):
    """(dlogs k_i, standard-form Jacobian limbs of k_i*G): k_i < 2^253, non-zero."""
    from gosnark_b200._lib import limbs_to_ints
    from gosnark_b200.synthetic import mint_points, rand_limbs
    ks = rand_limbs(n, seed)
    ks[:, 0] |= np.uint64(1)
    return limbs_to_ints(ks), mint_points(g, ks)


def load_set(g, pts, mode=0):
    from gosnark_b200 import bn128
    bs = bn128.BaseSet(g, limbs=pts, acc_mode=mode)
    if mode:
        assert bs.acc_mode() == mode
    return bs


def msm_device(L, bs, d_s, n, mont, d_out, stream=None):
    """b200_msm_device on `stream` (None: the library's stream); returns the C return code."""
    return L.b200_msm_device(bs.handle, None if d_s is None else d_s.data_ptr(), n, mont, d_out.data_ptr(),
                             None if stream is None else stream.cuda_stream)


def wait(stream):
    import torch
    if stream is None:
        torch.cuda.synchronize()        # the library's stream is not ordered with any torch stream
    else:
        stream.synchronize()


def sum_partials(L, g, d_recs, count, stream=None):
    from gosnark_b200._lib import check, ptr
    out = np.zeros(WORDS[g], np.uint64)
    fn = L.b200_g1_sum_partials if g == 1 else L.b200_g2_sum_partials
    check(fn(d_recs.data_ptr(), count, ptr(out), None if stream is None else stream.cuda_stream))
    return unflatten(g, out)[0]


SIZES = {1: 1 << 14, 2: 1 << 11}     # the sizes of test_gpu_msm.py's known-discrete-log tests


@pytest.fixture(scope="module")
def sets(lib):
    """(group, acc mode) -> (dlogs, base set) at SIZES, minted once per group."""
    made, minted = {}, {}

    def get(g, mode):
        if g not in minted:
            minted[g] = mint(g, SIZES[g], 0xD0 + g)
        if (g, mode) not in made:
            made[(g, mode)] = (minted[g][0], load_set(g, minted[g][1], mode))
        return made[(g, mode)]
    yield get
    for _, bs in made.values():
        bs.free()


def scalar_vectors(n, rng):
    """name -> n scalars < r: full width with 0 / 1 / r-1 mixed in, small (< 2^16, witness-like), all 0, all 1, all r-1."""
    full = [rng.randrange(R) for _ in range(n)]
    for i, v in zip(rng.sample(range(n), 9), (0, 0, 0, 1, 1, 1, R - 1, R - 1, R - 1)):
        full[i] = v
    return {"full": full, "small": [rng.randrange(1 << 16) for _ in range(n)], "zero": [0] * n, "one": [1] * n,
            "r-1": [R - 1] * n}


def to_mont_limbs(ss):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs([s * MONT % R for s in ss])


# ---- b200_msm_device ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g", [1, 2])
def test_msm_device_known_discrete_logs(lib, sets, g, mode):
    """Standard-form scalars (scalars_mont = 0) and the same scalars uploaded as s*2^256 mod r (scalars_mont = 1) give
    the same record, (sum s_i k_i)*G, on the library's stream and on a torch side stream, under both accumulation
    kernels."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs
    ks, bs = sets(g, mode)
    n = len(ks)
    rng = random.Random(31 * g + mode)
    d_out = torch.zeros(REC_WORDS[g], dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    for name, ss in scalar_vectors(n, rng).items():
        exp = expect_affine(g, sum(k * s for k, s in zip(ks, ss)))
        for mont, limbs in ((0, ints_to_limbs(ss)), (1, to_mont_limbs(ss))):
            d_s = to_dev(limbs)
            for stream in (None, side):
                d_out.fill_(-1)
                torch.cuda.synchronize()
                check(msm_device(lib, bs, d_s, n, mont, d_out, stream))
                wait(stream)
                assert decode_record(g, from_dev(d_out)) == exp, (name, mont, stream)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g", [1, 2])
def test_msm_device_prefixes_and_size_bound(lib, sets, g, mode):
    """n = 0 (with and without a scalar pointer) is the infinity record — the reference's loop starts from (0,0,0);
    n = 1, a prefix and the whole set sum the first n terms; n beyond the set returns B200_EINVAL and leaves the set
    usable."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs
    ks, bs = sets(g, mode)
    n = len(ks)
    rng = random.Random(77 * g + mode)
    ss = [rng.randrange(R) for _ in range(n)]
    d_s = to_dev(ints_to_limbs(ss))
    d_out = torch.zeros(REC_WORDS[g], dtype=torch.int64, device="cuda")
    for use_ptr in (True, False):
        d_out.fill_(-1)
        torch.cuda.synchronize()
        check(msm_device(lib, bs, d_s if use_ptr else None, 0, 0, d_out))
        wait(None)
        assert decode_record(g, from_dev(d_out)) is None
    for m in (1, 2, n // 3 + 5, n - 1, n):
        d_out.fill_(-1)
        torch.cuda.synchronize()
        check(msm_device(lib, bs, d_s, m, 0, d_out))
        wait(None)
        assert decode_record(g, from_dev(d_out)) == expect_affine(g, sum(k * s for k, s in zip(ks[:m], ss[:m]))), m
    big = to_dev(ints_to_limbs(ss + [1]))
    assert msm_device(lib, bs, big, n + 1, 0, d_out) == EINVAL
    assert msm_device(lib, bs, big, n + 1, 1, d_out) == EINVAL
    check(msm_device(lib, bs, d_s, n, 0, d_out))
    wait(None)
    assert decode_record(g, from_dev(d_out)) == expect_affine(g, sum(k * s for k, s in zip(ks, ss)))


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("g,n", [(1, 3001), (2, 701)])
def test_index_range_shards_summed_by_sum_partials(lib, g, n, world):
    """bench.py's multi-GPU MSM on one GPU: `world` uneven contiguous slices [n*k//world, n*(k+1)//world), each its own
    base set and b200_msm_device call on alternating streams; the records, laid end to end as the all-gather leaves
    them, are added by b200_g*_sum_partials(count = world) into the whole MSM."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs
    ks, pts = mint(g, n, 0xE0 + g)
    rng = random.Random(1000 * g + world)
    ss = [rng.randrange(R) for _ in range(n)]
    ss[0], ss[n // 2], ss[n - 1] = 0, 1, R - 1
    d_s = to_dev(ints_to_limbs(ss))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    bounds = [(n * k // world, n * (k + 1) // world) for k in range(world)]
    sets_, recs = [], []
    try:
        for k, (lo, hi) in enumerate(bounds):
            sets_.append(load_set(g, pts[lo:hi]))
            recs.append(torch.full((REC_WORDS[g],), -1, dtype=torch.int64, device="cuda"))
        torch.cuda.synchronize()
        for k, (lo, hi) in enumerate(bounds):
            check(msm_device(lib, sets_[k], d_s[4 * lo:], hi - lo, 0, recs[k], streams[k % 2]))
        for st in streams:
            st.synchronize()
        gathered = torch.cat(recs)
        for k, (lo, hi) in enumerate(bounds):
            got = decode_record(g, from_dev(recs[k]))
            assert got == expect_affine(g, sum(a * b for a, b in zip(ks[lo:hi], ss[lo:hi]))), k
        assert sum_partials(lib, g, gathered, world) == expect_out(g, sum(a * b for a, b in zip(ks, ss)))
    finally:
        for bs in sets_:
            bs.free()


# ---- b200_g*_sum_partials on records built here ------------------------------------------------------------------
POOL = 4096


@pytest.fixture(scope="module")
def pools(lib):
    """group -> (dlogs, affine points) of POOL + 1 distinct minted points."""
    made = {}

    def get(g):
        if g not in made:
            ks, pts = mint(g, POOL + 1, 0xF0 + g)
            made[g] = (ks, [tuple(OG[g].affine(p)[:2]) for p in unflatten(g, pts)])
        return made[g]
    return get


def build_records(g, pool, count, rng):
    """`count` records: distinct points, all-zero infinity records, the same point again under another z (the sum
    must double it), and negations of earlier points (the sum must cancel them).  Returns (records, expected dlog)."""
    ks, aff = pool
    recs, chosen, total = [], [], 0
    for i in range(count):
        u = rng.random()
        if i == 1 or (chosen and u < 0.12):           # an earlier point again: record 1 always repeats record 0
            j = chosen[0] if i == 1 else rng.choice(chosen)
            xy, k = aff[j], ks[j]
        elif chosen and u < 0.24:                     # the negation of an earlier point
            j = rng.choice(chosen)
            xy, k = neg_affine(g, aff[j]), -ks[j]
        elif u < 0.32 and i > 1:
            xy, k = None, 0
        else:
            j = i % len(ks)
            chosen.append(j)
            xy, k = aff[j], ks[j]
        recs.append(encode_record(g, xy, rand_z(g, rng)))
        total += k
    return np.stack(recs), total


@pytest.mark.parametrize("count", [1, 2, 3, 31, 32, 33, 255, 256, 257, 1000, 4097])
@pytest.mark.parametrize("g", [1, 2])
def test_sum_partials_mixed_records(lib, pools, g, count):
    """Counts around the 32-lane shuffle tree and the 256-thread block of k_sum_points, with infinity records, repeated
    points and cancelling pairs mixed in; the built records themselves decode to the points they were built from."""
    rng = random.Random(count * 7 + g)
    recs, total = build_records(g, pools(g), count, rng)
    assert decode_record(g, recs[0]) == pools(g)[1][0]
    assert sum_partials(lib, g, to_dev(recs), count) == expect_out(g, total)


@pytest.mark.parametrize("count,where", [(2, (0, 1)), (33, (0, 32)), (257, (0, 256)), (300, (37, 293))])
@pytest.mark.parametrize("g", [1, 2])
def test_sum_partials_double_and_cancel_at_each_level(lib, pools, g, count, where):
    """Only two finite records, everything else infinity: P under two different z must give 2P, P with -P the all-zero
    infinity.  The positions meet in the last shuffle step (0, 1), in the fold of the warp sums (0, 32) and in one
    thread's strided accumulation (0, 256), (37, 293).  The reference's P + P -> infinity (SURVEY H6) does not apply."""
    ks, aff = pools(g)
    rng = random.Random(count + 11 * g)
    for sign in (1, -1):
        recs = np.zeros((count, REC_WORDS[g]), np.uint64)
        recs[where[0]] = encode_record(g, aff[5], rand_z(g, rng))
        recs[where[1]] = encode_record(g, aff[5] if sign > 0 else neg_affine(g, aff[5]), rand_z(g, rng))
        assert sum_partials(lib, g, to_dev(recs), count) == expect_out(g, ks[5] * (1 + sign)), sign


@pytest.mark.parametrize("count", [2, 64, 513, 4096])
@pytest.mark.parametrize("g", [1, 2])
def test_sum_partials_total_infinity(lib, pools, g, count):
    """A set whose total is the point at infinity (pairs P, -P in shuffled order; an odd count adds one infinity
    record) comes out all-zero: x, y and z."""
    ks, aff = pools(g)
    rng = random.Random(5 * count + g)
    half = count // 2
    recs = [encode_record(g, aff[i], rand_z(g, rng)) for i in range(half)]
    recs += [encode_record(g, neg_affine(g, aff[i]), rand_z(g, rng)) for i in range(half)]
    recs += [encode_record(g, None, None)] * (count % 2)
    order = list(range(count))
    rng.shuffle(order)
    got = sum_partials(lib, g, to_dev(np.stack([recs[i] for i in order])), count)
    assert got == expect_out(g, 0)
    flat = got if g == 1 else [c for pair in got for c in pair]
    assert all(c == 0 for c in flat)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("g", [1, 2])
def test_sum_partials_documented_maximum(lib, pools, g):
    """count = 2^20, the documented maximum: 4096 distinct records tiled 256 times sum to 256 times their sum."""
    ks, aff = pools(g)
    rng = random.Random(99 + g)
    base = np.stack([encode_record(g, aff[i], rand_z(g, rng)) for i in range(POOL)])
    total = sum(ks[:POOL])
    d = to_dev(np.tile(base, (256, 1)))
    assert sum_partials(lib, g, d, 1 << 20) == expect_out(g, 256 * total)
    assert sum_partials(lib, g, d, POOL) == expect_out(g, total)


@pytest.mark.parametrize("g", [1, 2])
def test_sum_partials_bad_arguments(lib, pools, g):
    """count = 0, count = 2^20 + 1 and null pointers return B200_EINVAL; valid calls still work afterwards."""
    from gosnark_b200._lib import ptr
    ks, aff = pools(g)
    rec = to_dev(encode_record(g, aff[0], 7 if g == 1 else (7, 3)))
    out = np.zeros(WORDS[g], np.uint64)
    fn = lib.b200_g1_sum_partials if g == 1 else lib.b200_g2_sum_partials
    assert fn(rec.data_ptr(), 0, ptr(out), None) == EINVAL
    assert fn(rec.data_ptr(), (1 << 20) + 1, ptr(out), None) == EINVAL
    assert fn(None, 1, ptr(out), None) == EINVAL
    assert fn(rec.data_ptr(), 1, None, None) == EINVAL
    assert sum_partials(lib, g, rec, 1) == expect_out(g, ks[0])


# ---- out-of-range inputs on the _device entry points --------------------------------------------------------------
def poly_mul_checked(L, rng):
    """A valid b200_poly_mul must succeed and give the schoolbook product."""
    from gosnark_b200._lib import check, ints_to_limbs, limbs_to_ints, ptr
    a = [rng.randrange(R) for _ in range(5)]
    b = [rng.randrange(R) for _ in range(4)]
    out = np.zeros((8, 4), np.uint64)
    check(L.b200_poly_mul(ptr(ints_to_limbs(a)), 5, ptr(ints_to_limbs(b)), 4, ptr(out)))
    exp = [0] * 8
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            exp[i + j] = (exp[i + j] + x * y) % R
    assert limbs_to_ints(out) == exp


@pytest.mark.parametrize("g", [1, 2])
def test_out_of_range_scalar_on_msm_device_is_read_as_zero_and_not_reported(lib, g):
    """b200_msm_device with scalars_mont = 0 and scalars r and 2^256 - 1 returns B200_OK and sums them as 0.  Nothing
    reports them later: a following valid b200_g*_msm on the same set, and a valid b200_poly_mul, succeed with the
    right values (a stale device error flag would fail them with B200_ERANGE).  With scalars_mont = 1 nothing is
    range-checked: any 256-bit v is read as v * 2^-256 mod r.  The host-pointer b200_g*_msm still rejects r."""
    import torch
    from gosnark_b200._lib import B200Error, check, ints_to_limbs
    n = 64
    ks, pts = mint(g, n, 0xA0 + g)
    bs = load_set(g, pts)
    rng = random.Random(3 + g)
    try:
        ss = [rng.randrange(R) for _ in range(n)]
        bad = ints_to_limbs(ss)
        bad[3] = ints_to_limbs([R])[0]
        bad[40] = ints_to_limbs([(1 << 256) - 1])[0]
        as_read = [0 if i in (3, 40) else s for i, s in enumerate(ss)]
        d_out = torch.zeros(REC_WORDS[g], dtype=torch.int64, device="cuda")
        for follow_up in ("msm", "poly_mul"):
            for stream in (None, torch.cuda.Stream()):
                check(msm_device(lib, bs, to_dev(bad), n, 0, d_out, stream))
                wait(stream)
                assert decode_record(g, from_dev(d_out)) == expect_affine(g, sum(k * s for k, s in zip(ks, as_read)))
            if follow_up == "msm":
                assert bs.msm(ss) == expect_out(g, sum(k * s for k, s in zip(ks, ss)))
            else:
                poly_mul_checked(lib, rng)
        mont = [s * MONT % R for s in ss]
        mont[3] += R                                   # same residue, not reduced
        mont[40] = (1 << 256) - 1
        check(msm_device(lib, bs, to_dev(ints_to_limbs(mont)), n, 1, d_out))
        wait(None)
        mont_inv = pow(MONT, -1, R)
        assert decode_record(g, from_dev(d_out)) == expect_affine(g, sum(k * v * mont_inv for k, v in zip(ks, mont)))
        assert bs.msm(ss) == expect_out(g, sum(k * s for k, s in zip(ks, ss)))
        with pytest.raises(B200Error) as e:
            bs.msm(limbs=bad)
        assert e.value.code == -4
        assert bs.msm(ss) == expect_out(g, sum(k * s for k, s in zip(ks, ss)))
    finally:
        bs.free()


@pytest.fixture(scope="module")
def groth(lib):
    from gosnark_b200._lib import check
    from gosnark_b200.synthetic import SyntheticGroth16
    syn = SyntheticGroth16(10)
    pk = syn.load_pk()
    yield syn, pk
    check(lib.b200_pk_free(pk))


def monomial_quotient(e, z):
    """Quotient of x^e by the monic polynomial z (coefficients mod r, low to high)."""
    d = len(z) - 1
    rem = [0] * (e + 1)
    rem[e] = 1
    q = [0] * (e - d + 1)
    for i in range(e, d - 1, -1):
        c = rem[i]
        if c:
            q[i - d] = c
            for j in range(d + 1):
                rem[i - d + j] = (rem[i - d + j] - c * z[j]) % R
    return q


def check_proof(g1g2_words, exp):
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    G1, G2 = o.BN.G1, o.BN.G2
    pa, pc = _unflatten_g1(g1g2_words[:24])
    pb = _unflatten_g2(g1g2_words[24:])[0]
    ea, eb, ec = exp
    assert G1.affine(pa) == G1.affine(G1.mul_scalar(G1.G, ea))
    assert G2.affine(pb) == G2.affine(G2.mul_scalar(G2.G, eb))
    assert G1.affine(pc) == G1.affine(G1.mul_scalar(G1.G, ec))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("what", ["witness", "px"])
def test_out_of_range_input_on_prove_device_is_read_as_zero_and_not_reported(lib, groth, what):
    """b200_groth16_prove_device with one witness entry >= r, or one coefficient >= r in the top part of px (the part
    the division reads), returns B200_OK and proves as if that value were 0; the next valid b200_groth16_prove on the
    same key returns the known-discrete-log proof instead of a stale B200_ERANGE."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, limbs_to_ints, ptr
    syn, pk = groth
    w, px = syn.w.copy(), syn.px.copy()
    saved = syn.w, syn.h0
    try:
        if what == "witness":
            j = syn.npublic + 3                       # feeds A, B and C
            w[j] = ints_to_limbs([R])[0]
            syn.w = syn.w.copy()
            syn.w[j] = 0
        else:
            j = syn.n + 2                             # px[n..2n-2] fix the quotient by Z (degree n)
            px[j] = ints_to_limbs([(1 << 256) - 1])[0]
            c = limbs_to_ints(syn.px[j:j + 1])[0]
            h = limbs_to_ints(syn.h0)
            for i, qi in enumerate(monomial_quotient(j, limbs_to_ints(syn.z))):
                h[i] = (h[i] - c * qi) % R
            syn.h0 = ints_to_limbs(h)
        exp_bad = syn.expected_dlogs()
    finally:
        syn.w, syn.h0 = saved
    rr, ss = ints_to_limbs([syn.r]), ints_to_limbs([syn.s])
    d_w, d_px = to_dev(w), to_dev(px)
    d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
    for stream in (None, torch.cuda.Stream()):
        check(lib.b200_groth16_prove_device(pk, d_w.data_ptr(), syn.m, d_px.data_ptr(), px.shape[0], ptr(rr), ptr(ss),
                                            d_out.data_ptr(), None if stream is None else stream.cuda_stream))
        wait(stream)
        check_proof(from_dev(d_out), exp_bad)
        pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
        check(lib.b200_groth16_prove(pk, ptr(syn.w), syn.m, ptr(syn.px), syn.px.shape[0], ptr(rr), ptr(ss), ptr(pa),
                                     ptr(pb), ptr(pc)))
        check_proof(np.concatenate([pa, pc, pb]), syn.expected_dlogs())
