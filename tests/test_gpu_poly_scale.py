"""GPU: the F_r polynomial engine (ntt.cuh / poly_host.cuh behind b200_poly_mul, b200_poly_div, b200_poly_eval) at every
transform shape it takes, against exact Python-int references.

The transform path changes with log2 of the size: per-stage kernels below 2^10, one contiguous fused pass at 2^10, one
strided pass then the contiguous one from 2^11 to 2^18, two strided passes from 2^19 and three at 2^27, the product cap.
So products are taken at lo = len(a) + len(b) - 1 = 2^k and 2^k + 1 around each switch, and divisions at quotient lengths
2^k and 2^k + 1 with divisors far shorter and far longer than the quotient (the Newton inverse then loads len(b) or 2P
divisor terms per doubling).  Random operands are checked by evaluation at random points (O(n) per check; a wrong output
passes with probability about deg / r); structured operands are compared coefficient by coefficient."""
import os
import random

import numpy as np
import pytest

from fr_ref import R, R_LIMBS, from_ints, horner, r_minus, rand_limbs, small_limbs, to_ints

pytestmark = pytest.mark.gpu
EINVAL, ERANGE, EDIVZERO = -3, -4, -5


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


def mul(L, a, b):
    from gosnark_b200._lib import check, ptr
    out = np.zeros((a.shape[0] + b.shape[0] - 1, 4), dtype=np.uint64)
    check(L.b200_poly_mul(ptr(a), a.shape[0], ptr(b), b.shape[0], ptr(out)))
    return out


def div(L, a, b, with_rem=True):
    from gosnark_b200._lib import check, ptr
    q = np.zeros((a.shape[0] - b.shape[0] + 1, 4), dtype=np.uint64)
    rem = np.zeros((max(b.shape[0] - 1, 1), 4), dtype=np.uint64)
    check(L.b200_poly_div(ptr(a), a.shape[0], ptr(b), b.shape[0], ptr(q), ptr(rem) if with_rem else None))
    return q, rem[: b.shape[0] - 1]


def taus(seed, count):
    rng = random.Random(seed)
    return [rng.randrange(R) for _ in range(count)]


def check_product(a, b, out, seed):
    """out(tau) == a(tau) * b(tau) at two random tau (one above 2^20 coefficients: the Python check is the cost)."""
    ai, bi, oi = to_ints(a), to_ints(b), to_ints(out)
    for t in taus(seed, 1 if len(oi) > (1 << 20) else 2):
        assert horner(oi, t) == horner(ai, t) * horner(bi, t) % R, (len(ai), len(bi), t)


def check_division(a, b, q, rem, seed):
    """a(tau) == q(tau) b(tau) + rem(tau) at independent random tau, with len(q) = na - nb + 1 and len(rem) = nb - 1: by
    uniqueness of division a complete check up to a failure probability of about 2 deg / r."""
    assert q.shape[0] == a.shape[0] - b.shape[0] + 1 and rem.shape[0] == b.shape[0] - 1
    ai, bi, qi, ri = to_ints(a), to_ints(b), to_ints(q), to_ints(rem)
    for t in taus(seed, 1 if len(ai) > (1 << 20) else 2):
        assert horner(ai, t) == (horner(qi, t) * horner(bi, t) + horner(ri, t)) % R, (len(ai), len(bi), t)


PRODUCT_K = [9, 10, 11, 18, 19, 22]
PRODUCT_LO = [lo for k in PRODUCT_K for lo in (1 << k, (1 << k) + 1)]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("shape", ["unequal", "len1"])
@pytest.mark.parametrize("lo", PRODUCT_LO)
def test_mul_random(L, lo, shape):
    """Full-range random factors, na != nb or one factor of length 1, checked by evaluation."""
    na = lo // 3 + 1 if shape == "unequal" else lo
    nb = lo - na + 1
    a, b = rand_limbs(na, lo), rand_limbs(nb, lo + 1)
    check_product(a, b, mul(L, a, b), lo)


def trapezoid(na, nb):
    k = np.arange(na + nb - 1, dtype=np.int64)
    return np.minimum.reduce([k, np.full_like(k, na - 1), np.full_like(k, nb - 1), na + nb - 2 - k]) + 1


def check_structured(L, na, nb, seed):
    lo = na + nb - 1
    rng = random.Random(seed)
    # a * x^(nb-1): the shift of a full-range a
    a = rand_limbs(na, seed)
    e = np.zeros((nb, 4), dtype=np.uint64)
    e[nb - 1, 0] = 1
    out = mul(L, a, e)
    assert not out[: nb - 1].any() and np.array_equal(out[nb - 1:], a), "shift"
    # all-ones x all-ones: the trapezoid; all-(r-1) x all-ones: r - trapezoid (every coefficient at the reduction edge)
    t = trapezoid(na, nb)
    ones_a, ones_b = small_limbs(np.ones(na, dtype=np.uint64)), small_limbs(np.ones(nb, dtype=np.uint64))
    assert np.array_equal(mul(L, ones_a, ones_b), small_limbs(t)), "trapezoid"
    del ones_a
    assert np.array_equal(mul(L, r_minus(np.ones(na, dtype=np.uint64)), ones_b), r_minus(t)), "r - trapezoid"
    del ones_b, t
    # one full-range non-zero at the last index of each operand: u v at index lo - 1, zero elsewhere
    u, v = rng.randrange(R), rng.randrange(R)
    a = np.zeros((na, 4), dtype=np.uint64)
    b = np.zeros((nb, 4), dtype=np.uint64)
    a[na - 1], b[nb - 1] = from_ints([u])[0], from_ints([v])[0]
    out = mul(L, a, b)
    assert not out[: lo - 1].any() and to_ints(out[lo - 1:]) == [u * v % R], "last-index product"


@pytest.mark.timeout(900)
@pytest.mark.parametrize("lo", PRODUCT_LO)
def test_mul_structured(L, lo):
    """Whole outputs compared exactly: shift, trapezoid, r - trapezoid, last-index product (na != nb)."""
    na = lo // 3 + 1
    check_structured(L, na, lo - na + 1, lo)


def host_bytes_free():
    try:
        return os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    except (ValueError, OSError):
        return 0


@pytest.mark.timeout(1200)
def test_mul_cap_2_27(L):
    """lo = 2^27, the product cap: three strided passes, the last with k = 1 (512 columns, two tiles per group).  Only
    structured inputs (the Python check of a random product would take minutes); lo = 2^27 + 1 is refused."""
    from gosnark_b200._lib import ptr
    one = np.zeros((1, 4), dtype=np.uint64)
    half = 1 << 26
    assert L.b200_poly_mul(ptr(one), half + 1, ptr(one), half + 1, ptr(one)) == EINVAL   # refused before any read
    need = 20 << 30
    if host_bytes_free() < need:
        pytest.skip(f"the 2^27-coefficient product needs about 20 GB of free host memory (have {host_bytes_free() >> 30} GB)")
    check_structured(L, half, half + 1, 27)


DIV_K = [9, 10, 18, 19, 21]
# (nq, nb, monic): a divisor far shorter than the quotient and one far longer, monic and not on both sides
DIV_CASES = [(nq, nb, monic) for k in DIV_K for nq, flip in (((1 << k), 0), ((1 << k) + 1, 1))
             for nb, monic in ((5, bool(flip)), (2 * nq + 3, not flip))]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("nq,nb,monic", DIV_CASES, ids=[f"nq{q}-nb{b}-{'monic' if m else 'nonmonic'}" for q, b, m in DIV_CASES])
def test_div(L, nq, nb, monic):
    na = nq + nb - 1
    a, b = rand_limbs(na, na), rand_limbs(nb, nb)
    if monic:
        b[nb - 1] = (1, 0, 0, 0)
    else:
        b[nb - 1, 0] |= np.uint64(1)          # non-zero leading coefficient
    q, rem = div(L, a, b)
    check_division(a, b, q, rem, na + nb)


def test_div_zero_leading_coefficient_large(L):
    """A divisor whose leading coefficient is 0 at 2^19 + 1 coefficients: EDIVZERO (the reference's ModInverse(0) panic);
    the next division is right."""
    from gosnark_b200._lib import B200Error
    nb = (1 << 19) + 1
    b = rand_limbs(nb, 3)
    b[nb - 1] = 0
    with pytest.raises(B200Error) as e:
        div(L, rand_limbs(nb + 100, 4), b)
    assert e.value.code == EDIVZERO
    a, b = rand_limbs(40, 5), rand_limbs(7, 6)
    q, rem = div(L, a, b)
    check_division(a, b, q, rem, 7)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [(1 << 20) + 1, 1 << 21])
def test_divisor_polynomial_by_zero_poly(L, n):
    """DivisorPolynomial(px, Z) with Z = b200_zero_poly(n) and px = h Z + rem minted in Python (h with a few full-range
    terms spread over its n - 1 coefficients, the first and last included; rem dense, deg < n): the quotient is h and the
    remainder rem, coefficient for coefficient, with and without the remainder requested."""
    from gosnark_b200._lib import check, ptr
    z = np.zeros((n + 1, 4), dtype=np.uint64)
    check(L.b200_zero_poly(n, ptr(z)))
    zi = to_ints(z)
    rng = random.Random(n)
    terms = {0: rng.randrange(1, R), n - 2: rng.randrange(1, R)}
    for k in rng.sample(range(1, n - 2), 4):
        terms[k] = rng.randrange(1, R)
    rem = rand_limbs(n, n)
    px = to_ints(rem) + [0] * (n - 1)
    for k, c in terms.items():
        for i, zc in enumerate(zi):
            px[k + i] += c * zc
    px = from_ints(px)
    h = np.zeros((n - 1, 4), dtype=np.uint64)
    for k, c in terms.items():
        h[k] = from_ints([c])[0]
    q, r = div(L, px, z)
    assert np.array_equal(q, h) and np.array_equal(r, rem)
    q2, _ = div(L, px, z, with_rem=False)
    assert np.array_equal(q2, h)


@pytest.mark.timeout(600)
def test_poly_eval_large(L):
    """b200_poly_eval and b200_poly_eval_batch at 2^20 + 3 coefficients against Horner, at a random x and at r - 1."""
    from gosnark_b200._lib import check, limbs_to_ints, ptr
    n = (1 << 20) + 3
    polys = rand_limbs(2 * n, 11)
    ints = to_ints(polys)
    for x in (taus(12, 1)[0], R - 1):
        X = from_ints([x])
        exp = [horner(ints[:n], x), horner(ints[n:], x)]
        out = np.zeros(4, dtype=np.uint64)
        check(L.b200_poly_eval(ptr(polys), n, ptr(X), ptr(out)))
        assert limbs_to_ints(out)[0] == exp[0]
        outb = np.zeros((2, 4), dtype=np.uint64)
        check(L.b200_poly_eval_batch(ptr(polys), 2, n, ptr(X), ptr(outb)))
        assert limbs_to_ints(outb) == exp


@pytest.mark.parametrize("where", ["mul-a", "mul-b", "div-a", "div-b"])
def test_coefficient_out_of_range(L, where):
    """A coefficient >= r at the last index of one input (2^19 + 1 coefficients) is refused with ERANGE, also when it is
    the divisor's leading coefficient; the next valid call is right, with no stale error flag."""
    from gosnark_b200._lib import B200Error
    n = (1 << 19) + 1
    a, b = rand_limbs(n, 21), rand_limbs(n if where.startswith("mul") else 1000, 22)
    (a if where.endswith("a") else b)[-1] = R_LIMBS
    with pytest.raises(B200Error) as e:
        mul(L, a, b) if where.startswith("mul") else div(L, a, b)
    assert e.value.code == ERANGE, e.value
    assert to_ints(mul(L, small_limbs([1, 2]), small_limbs([3]))) == [3, 6]
    a, b = rand_limbs(50, 23), rand_limbs(9, 24)
    q, rem = div(L, a, b)
    check_division(a, b, q, rem, 25)
