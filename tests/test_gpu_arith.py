"""The field, tower and curve arithmetic headers (fp.cuh, fp2.cuh, ec.cuh, pairing.cuh, pairing_warp.cuh, glv.cuh) ON THE
DEVICE, against the oracle, at their carry and reduction edges.

tests/test_host_arith.py runs these headers through the host carry-flag emulation; here tests/device/arith_device.cu
compiles them with nvcc for sm_90a, where the carry crosses statement boundaries through the condition-code register,
the hot kernels' force-inlined products (INL = true) differ from the cold kernels' outlined ones (INL = false), and the
warp code shuffles and shares memory for real.  Both vehicles run the edge vectors of tests/arith_edges.py: every edge
value also as its Montgomery preimage e * 2^-256 mod p, so that the limbs the carry chains see are the edges.

The second half feeds edge-valued coordinates straight into the product's element-wise entry points
(b200_g{1,2}_{add,double,neg,affine,mul}_batch, b200_fq12_mul_batch), which accept any triple of canonical coordinates,
and compares them X, Y, Z-exactly with the oracle's formulas, which are defined on any triple too."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

import arith_edges
import build as b200build
from oracle import ref_py as o

pytestmark = pytest.mark.gpu

Q, R = o.Q, o.R
F2, F12 = o.BN.Fq2, o.BN.Fq12
BULK = 1 << 20                    # random operand pairs per op and build variant
VARIANTS = [0, 1]                 # 0: outlined (__noinline__) products, 1: force-inlined (FqH / FrH / Fq2H)
_i, _vp, _sz = ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t
_SIGS = {
    "g_fp_op": [_i, _i, _i, _vp, _vp, _vp, _sz], "g_geq": [_i, _i, _vp, _vp, _sz], "g_mul_full": [_i, _vp, _vp, _vp, _sz],
    "g_redc_wide": [_i, _i, _vp, _vp, _sz], "g_fq2_op": [_i, _i, _vp, _vp, _vp, _sz],
    "g_g1_xyzz": [_i, _i, _vp, _vp, _vp, _sz], "g_g2_xyzz": [_i, _i, _vp, _vp, _vp, _sz],
    "g_g1_jac": [_i, _i, _vp, _vp, _vp, _sz], "g_g2_jac": [_i, _i, _vp, _vp, _vp, _sz],
    "g_f12_op": [_i, _vp, _vp, _vp, _sz], "g_f12_warp": [_i, _vp, _vp, _vp, _sz],
    "g_glv_mul": [_vp, _vp, _vp, _sz], "g_pairing": [_i, _vp, _vp, _vp, _sz],
}


@pytest.fixture(scope="module")
def lib():
    L = ctypes.CDLL(b200build.build_gpu_arith())
    for name, args in _SIGS.items():
        getattr(L, name).argtypes = args
        getattr(L, name).restype = ctypes.c_int
    return L


# ---- marshalling ------------------------------------------------------------------------------------------------------
def pack(vals, nbytes=32):
    return np.frombuffer(b"".join(int(v).to_bytes(nbytes, "little") for v in vals), dtype=np.uint32).copy()


def unpack(words):
    """(n, k) uint32 rows -> list of ints (k limbs each)."""
    raw = np.ascontiguousarray(words).tobytes()
    w = 4 * words.shape[1]
    return [int.from_bytes(raw[i:i + w], "little") for i in range(0, len(raw), w)]


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def flat(xs):
    """nested tuples of ints (field elements, points, F_q^12) -> flat list of ints"""
    out = []
    for x in xs:
        if isinstance(x, tuple):
            out.extend(flat(x))
        else:
            out.append(x)
    return out


def expect_rows(got, expected, what, operands):
    """got: (n, k) uint32; expected: list of n ints of k limbs.  Reports the first mismatching operands."""
    exp = pack(expected, 4 * got.shape[1]).reshape(got.shape)
    bad = np.nonzero((got != exp).any(axis=1))[0]
    assert bad.size == 0, f"{what}: {bad.size} of {len(expected)} wrong, first at {[operands(int(i)) for i in bad[:3]]}"


def fp_op(lib, field, inl, op, A, B):
    n = len(A)
    out = np.zeros((n, 9), dtype=np.uint32)
    assert lib.g_fp_op(field, inl, op, ptr(pack(A)), ptr(pack(B)), ptr(out), n) == 0
    bad = np.nonzero(out[:, 8])[0]
    assert bad.size == 0, f"op {op}: Montgomery result >= p for {[(hex(A[i]), hex(B[i])) for i in bad[:3]]}"
    return out[:, :8]


def fq2_op(lib, inl, op, A, B):
    n = len(A)
    out = np.zeros((n, 17), dtype=np.uint32)
    assert lib.g_fq2_op(inl, op, ptr(pack(flat(A))), ptr(pack(flat(B))), ptr(out), n) == 0
    bad = np.nonzero(out[:, 16])[0]
    assert bad.size == 0, f"op {op}: Montgomery component >= p for {[(A[i], B[i]) for i in bad[:3]]}"
    return out[:, :16]


def f2_rows(rows):
    """(n, 16) -> list of (c0, c1)"""
    v = unpack(rows.reshape(-1, 8))
    return [(v[2 * i], v[2 * i + 1]) for i in range(len(v) // 2)]


# ---- F_q and F_r -----------------------------------------------------------------------------------------------------
FIELDS = [(0, Q), (1, R)]


def _binary_checks(lib, field, inl, p, A, B, tag):
    ops = lambda i: (hex(A[i]), hex(B[i]))
    expect_rows(fp_op(lib, field, inl, 0, A, B), [(a + b) % p for a, b in zip(A, B)], f"{tag} add", ops)
    expect_rows(fp_op(lib, field, inl, 1, A, B), [(a - b) % p for a, b in zip(A, B)], f"{tag} sub", ops)
    expect_rows(fp_op(lib, field, inl, 2, A, B), [a * b % p for a, b in zip(A, B)], f"{tag} mul", ops)


def _unary_checks(lib, field, inl, p, A, tag):
    ops = lambda i: hex(A[i])
    expect_rows(fp_op(lib, field, inl, 4, A, A), [(-a) % p for a in A], f"{tag} neg", ops)
    expect_rows(fp_op(lib, field, inl, 5, A, A), [a * a % p for a in A], f"{tag} sqr", ops)
    for op in (3, 6):                  # Fermat and binary-Euclid inversion: a * a^-1 == 1, 0 -> 0
        got = unpack(fp_op(lib, field, inl, op, A, A))
        bad = [i for i, (a, g) in enumerate(zip(A, got)) if (a * g % p != 1 if a else g != 0) or g >= p]
        assert not bad, f"{tag} inverse op {op}: wrong for {[hex(A[i]) for i in bad[:3]]}"


@pytest.mark.parametrize("inl", VARIANTS, ids=["outlined", "inlined"])
@pytest.mark.parametrize("field,p", FIELDS, ids=["Fq", "Fr"])
def test_fp_edge_pairs(lib, field, p, inl):
    """Every ordered pair of the edge set through add, sub and mul, every edge through neg, sqr and both inversions, and
    geq_modulus on the edges (all < p) and at and above p — each in one launch."""
    E = arith_edges.edges(p)
    A = [a for a in E for _ in E]
    B = [b for _ in E for b in E]
    _binary_checks(lib, field, inl, p, A, B, "edge")
    _unary_checks(lib, field, inl, p, E, "edge")
    over = [p, p + 1, p + 2, p + (1 << 32), p | 0xffffffff, (1 << 255), (1 << 256) - 1, (1 << 256) - 2]
    vals = E + over
    out = np.zeros(len(vals), dtype=np.int32)
    assert lib.g_geq(field, inl, ptr(pack(vals)), ptr(out), len(vals)) == 0
    assert list(out) == [0] * len(E) + [1] * len(over)


_RAND = {}


def _random_operands(p):
    if p not in _RAND:
        rng = random.Random(p & 0xffff)
        _RAND[p] = ([rng.randrange(p) for _ in range(BULK)], [rng.randrange(p) for _ in range(BULK)])
    return _RAND[p]


@pytest.mark.parametrize("inl", VARIANTS, ids=["outlined", "inlined"])
@pytest.mark.parametrize("field,p", FIELDS, ids=["Fq", "Fr"])
def test_fp_bulk(lib, field, p, inl):
    """2^20 random pairs per op in one launch each: add, sub, mul, neg, sqr, inverse, inverse_vartime."""
    A, B = _random_operands(p)
    _binary_checks(lib, field, inl, p, A, B, "bulk")
    _unary_checks(lib, field, inl, p, A, "bulk")


@pytest.mark.parametrize("inl", VARIANTS, ids=["outlined", "inlined"])
def test_wide_product_and_reduction(lib, inl):
    """mul_full on every pair of the wide edges (up to (2^256 - 1)^2) and 2^20 random 256-bit pairs; redc_wide on the
    reduction edges (up to t = p * 2^256 - 1) and 2^20 random t < p * 2^256, for both moduli."""
    W = arith_edges.wide_edges()
    rng = random.Random(77)
    A = [a for a in W for _ in W] + [rng.getrandbits(256) for _ in range(BULK)]
    B = [b for _ in W for b in W] + [rng.getrandbits(256) for _ in range(BULK)]
    out = np.zeros((len(A), 16), dtype=np.uint32)
    assert lib.g_mul_full(inl, ptr(pack(A)), ptr(pack(B)), ptr(out), len(A)) == 0
    expect_rows(out, [a * b for a, b in zip(A, B)], "mul_full", lambda i: (hex(A[i]), hex(B[i])))
    for field, p in FIELDS:
        rinv = pow(1 << 256, -1, p)
        T = arith_edges.redc_edges(p) + [rng.randrange(p << 256) for _ in range(BULK)]
        out = np.zeros((len(T), 8), dtype=np.uint32)
        assert lib.g_redc_wide(field, inl, ptr(pack(T, 64)), ptr(out), len(T)) == 0
        expect_rows(out, [t * rinv % p for t in T], f"redc_wide field {field}", lambda i: hex(T[i]))


# ---- F_q^2 -----------------------------------------------------------------------------------------------------------
def _fq2_checks(lib, inl, A, B, tag, inverses=True):
    ops = lambda i: (A[i], B[i])
    for op, fn in ((0, lambda a, b: F2.add(a, b)), (1, lambda a, b: F2.sub(a, b)), (2, lambda a, b: F2.mul(a, b)),
                   (4, lambda a, b: F2.square(a)), (5, lambda a, b: F2.neg(a))):
        got = f2_rows(fq2_op(lib, inl, op, A, B))
        bad = [i for i, (a, b, g) in enumerate(zip(A, B, got)) if g != fn(a, b)]
        assert not bad, f"{tag} fq2 op {op}: {len(bad)} wrong, first at {[ops(i) for i in bad[:3]]}"
    if inverses:
        for op in (3, 6):
            got = f2_rows(fq2_op(lib, inl, op, A, B))
            bad = [i for i, (a, g) in enumerate(zip(A, got)) if g != (F2.inverse(a) if a != (0, 0) else (0, 0))]
            assert not bad, f"{tag} fq2 inverse op {op}: wrong for {[A[i] for i in bad[:3]]}"


@pytest.mark.parametrize("inl", VARIANTS, ids=["outlined", "inlined"])
def test_fq2_edge_components(lib, inl):
    """F_q^2 ops with components from the edge set, including the lazy-reduction extremes of the product in Montgomery
    form: a0 b0 = 0 with a1 b1 maximal (representatives p - 1) and the reverse — v0 - v1 + p^2 near 0 and near 2 p^2."""
    E = arith_edges.edges(Q)
    m1 = arith_edges.montgomery_preimages(Q, [Q - 1])[0]
    rng = random.Random(21)
    A = [(0, m1)] * len(E) + [(m1, 0)] * len(E) + [(m1, m1)] * len(E)
    B = [(x, m1) for x in E] + [(m1, x) for x in E] + [(x, 0) for x in E]
    A += [(a0, a1) for a0 in E for a1 in E]                      # every component pair ...
    B += [(rng.choice(E), rng.choice(E)) for _ in range(len(E) ** 2)]   # ... times edge-valued partners
    _fq2_checks(lib, inl, A, B, "edge")


@pytest.mark.parametrize("inl", VARIANTS, ids=["outlined", "inlined"])
def test_fq2_bulk(lib, inl):
    """2^20 random F_q^2 products and squares in one launch each (sums, differences and inversions on 2^16)."""
    A0, B0 = _random_operands(Q)
    A = list(zip(A0[:BULK], B0[:BULK]))
    B = list(zip(B0[::-1], A0[::-1]))
    for op, fn in ((2, F2.mul), (4, lambda a, b: F2.square(a))):
        got = f2_rows(fq2_op(lib, inl, op, A, B))
        bad = [i for i, (a, b, g) in enumerate(zip(A, B, got)) if g != fn(a, b)]
        assert not bad, f"bulk fq2 op {op}: {len(bad)} wrong, first at {[(A[i], B[i]) for i in bad[:3]]}"
    _fq2_checks(lib, inl, A[:1 << 16], B[:1 << 16], "bulk")


# ---- curve formulas --------------------------------------------------------------------------------------------------
def _grp(gname):
    return (o.BN.G1, 1) if gname == "G1" else (o.BN.G2, 2)


def _edge_z(gname):
    """Z values of edge shape: 1, p - 1, and the Montgomery preimages 2^-256 (representative 1) and of p - 1."""
    zs = [1, Q - 1] + arith_edges.montgomery_preimages(Q, [1, Q - 1, (1 << 255) % Q])
    return zs if gname == "G1" else [(z, 0) for z in zs] + [(0, z) for z in zs[:2]] + [(zs[2], zs[3])]


def _rescale(G, P, z):
    """The same point with Jacobian Z multiplied by z."""
    F = G.F
    z2 = F.square(z)
    return (F.mul(P[0], z2), F.mul(P[1], F.mul(z2, z)), F.mul(P[2], z))


def _points(gname, seed, k):
    G, _ = _grp(gname)
    rng = random.Random(seed)
    pts = [G.mul_scalar(G.G, rng.randrange(1, R)) for _ in range(k)]
    aff = G.affine(pts[0])
    one = G.F.one()
    pts.append((aff[0], aff[1], one))
    pts += [_rescale(G, (aff[0], aff[1], one), z) for z in _edge_z(gname)]
    return pts


def _xyzz(G, P):
    zz = G.F.square(P[2])
    return (P[0], P[1], zz, G.F.mul(zz, P[2]))


def _aff(G, P, W):
    if G.is_zero(P):
        return (0, 0) if W == 1 else ((0, 0), (0, 0))
    a = G.affine(P)
    return (a[0], a[1])


@pytest.mark.parametrize("inl", VARIANTS, ids=["outlined", "inlined"])
@pytest.mark.parametrize("gname", ["G1", "G2"])
def test_xyzz_group_law(lib, gname, inl):
    """madd, add, dbl, the Jacobian round trip and both affine conversions against the oracle's group law (affine
    parity), on points with random and edge-valued Z, including P + P, P + (-P) and infinity on either side."""
    G, W = _grp(gname)
    fn = lib.g_g1_xyzz if W == 1 else lib.g_g2_xyzz
    zero = G.F.zero()
    inf_x = (zero, zero, zero, zero)
    pts = _points(gname, 7 + W, 6)
    cases = []                                                   # (op, xyzz a, affine-or-xyzz b, expected affine)
    for i, P in enumerate(pts):
        Qp = pts[(i + 1) % len(pts)]
        PX = _xyzz(G, P)
        s = G.add(P, Qp) if G.affine(P) != G.affine(Qp) else G.double(P)
        cases += [(0, PX, _aff(G, Qp, W) + (zero, zero), _aff(G, s, W)), (1, PX, _xyzz(G, Qp), _aff(G, s, W)),
                  (2, PX, PX, _aff(G, G.double(P), W)), (3, PX, PX, _aff(G, P, W)), (4, PX, PX, _aff(G, P, W)),
                  (0, PX, _aff(G, P, W) + (zero, zero), _aff(G, G.double(P), W)), (1, PX, PX, _aff(G, G.double(P), W)),
                  (0, PX, _aff(G, G.neg(P), W) + (zero, zero), _aff(G, G.zero3(), W)),
                  (1, PX, _xyzz(G, G.neg(P)), _aff(G, G.zero3(), W)),
                  (0, inf_x, _aff(G, P, W) + (zero, zero), _aff(G, P, W)), (0, PX, (zero,) * 4, _aff(G, P, W)),
                  (1, inf_x, PX, _aff(G, P, W)), (1, PX, inf_x, _aff(G, P, W)), (2, inf_x, inf_x, _aff(G, G.zero3(), W))]
    for op in range(5):
        sel = [c for c in cases if c[0] == op]
        n = len(sel)
        out = np.zeros((n, 16 * W), dtype=np.uint32)
        assert fn(inl, op, ptr(pack(flat([c[1] for c in sel]))), ptr(pack(flat([c[2] for c in sel]))), ptr(out), n) == 0
        got = unpack(out.reshape(-1, 8))
        for k, c in enumerate(sel):
            assert got[2 * W * k:2 * W * (k + 1)] == flat(c[3]), (gname, inl, op, k)


@pytest.mark.parametrize("inl", VARIANTS, ids=["outlined", "inlined"])
@pytest.mark.parametrize("gname", ["G1", "G2"])
def test_reference_formulas_exact_jacobian(lib, gname, inl):
    """jac_add_ref / jac_double_ref X, Y, Z-exactly against the oracle's restatement of the reference, on curve points
    with random and edge-valued Z and on 4096 arbitrary triples of edge-valued coordinates (the formulas are defined on
    any triple; Z = 0 returns the other operand, equal operands give the reference's Z3 = 0)."""
    G, W = _grp(gname)
    fn = lib.g_g1_jac if W == 1 else lib.g_g2_jac
    pts = _points(gname, 11 + W, 4) + [G.G, G.zero3()]
    E = arith_edges.edges(Q)
    rng = random.Random(31 + W)
    el = (lambda: rng.choice(E)) if W == 1 else (lambda: (rng.choice(E), rng.choice(E)))
    trip = [(el(), el(), el()) for _ in range(4096)]
    A = pts + [pts[(i + 1) % len(pts)] for i in range(len(pts))] + trip + trip[:64]
    B = [pts[(i + 1) % len(pts)] for i in range(len(pts))] + pts + trip[::-1] + trip[:64]
    n = len(A)
    for op, exp in ((0, [G.add(a, b) for a, b in zip(A, B)]), (1, [G.double(a) for a in A])):
        out = np.zeros((n, 24 * W), dtype=np.uint32)
        assert fn(inl, op, ptr(pack(flat(A))), ptr(pack(flat(B))), ptr(out), n) == 0
        got = unpack(out.reshape(-1, 8))
        bad = [k for k in range(n) if got[3 * W * k:3 * W * (k + 1)] != flat(exp[k])]
        assert not bad, (gname, inl, op, len(bad), [(A[k], B[k]) for k in bad[:2]])


# ---- F_q^12 ----------------------------------------------------------------------------------------------------------
def _f12(v):
    return tuple(tuple((v[6 * h + 2 * k], v[6 * h + 2 * k + 1]) for k in range(3)) for h in range(2))


def _f12_elems(k, seed):
    """k elements whose components are edge values (most) or random (every fourth)."""
    E = arith_edges.edges(Q)
    rng = random.Random(seed)
    out = []
    for i in range(k):
        pick = (lambda: rng.randrange(Q)) if i % 4 == 3 else (lambda: rng.choice(E))
        out.append(_f12([pick() for _ in range(12)]))
    return out


def _f12_run(fn, op, A, B):
    n = len(A)
    out = np.zeros((n, 96), dtype=np.uint32)
    assert fn(op, ptr(pack(flat(A))), ptr(pack(flat(B))), ptr(out), n) == 0
    v = unpack(out.reshape(-1, 8))
    return [_f12(v[12 * i:12 * (i + 1)]) for i in range(n)]


def test_f12_products_thread_and_warp(lib):
    """4096 products of edge-valued F_q^12 elements: the thread f12_mul / f12_sqr and the warp wp::f12_mul in each alias
    pattern (d != a != b, d = a, d = b, d = a = b) all equal the oracle."""
    n = 4096
    A, B = _f12_elems(n, 1), _f12_elems(n, 2)
    prod = [F12.mul(a, b) for a, b in zip(A, B)]
    sq = [F12.mul(a, a) for a in A]
    assert _f12_run(lib.g_f12_op, 5, A, B) == prod
    assert _f12_run(lib.g_f12_op, 6, A, B) == sq
    for op in (0, 1, 2):
        assert _f12_run(lib.g_f12_warp, op, A, B) == prod, op
    assert _f12_run(lib.g_f12_warp, 3, A, B) == sq


def test_f12_inverse_frobenius_exp_u(lib):
    """f12_inverse, f12_frobenius<1..3>, f12_exp_u and conjugation, thread and warp, against the oracle's plain
    exponentiations, on a few edge-valued elements (the oracle's exponentiations are slow)."""
    A = _f12_elems(12, 3) + [F12.one()]
    U = 4965661367192848881
    inv = [F12.inverse(a) for a in A]
    assert _f12_run(lib.g_f12_op, 0, A, A) == inv
    assert _f12_run(lib.g_f12_warp, 4, A, A) == inv
    fr = [A]
    for k in range(3):
        fr.append([F12.exp(x, Q) for x in fr[-1]])
    for k in (1, 2, 3):
        assert _f12_run(lib.g_f12_op, k, A, A) == fr[k], k
        assert _f12_run(lib.g_f12_warp, 4 + k, A, A) == fr[k], k
    few = A[:6]
    eu = [F12.exp(x, U) for x in few]
    assert _f12_run(lib.g_f12_op, 4, few, few) == eu
    assert _f12_run(lib.g_f12_warp, 8, few, few) == eu
    conj = [(a[0], tuple(F2.neg(c) for c in a[1])) for a in A]
    assert _f12_run(lib.g_f12_warp, 9, A, A) == conj


# ---- GLV and pairings ------------------------------------------------------------------------------------------------
def test_glv_half_warp_multiplication(lib):
    """glv_mul_halfwarp with scalars split by glv_decompose: the cases of the CPU emulation (edge scalars, random
    scalars, non-normalised points, infinity) plus points with edge-valued Z, an odd count (a half-warp with no
    product of its own), as group elements against the oracle."""
    G = o.BN.G1
    rng = random.Random(91)
    lam = 4407920970296243842393367215006156084916469457145843978461
    edge = [0, 1, 2, R - 1, R - 2, (1 << 128) - 1, 1 << 128, (1 << 128) + 1, 1 << 127, lam % R, (R - lam) % R, 1 << 253]
    ks = edge + [rng.randrange(R) for _ in range(12)]
    base = _points("G1", 5, 3) + [G.zero3()]
    pts = [base[i % len(base)] for i in range(len(ks))]
    ks.append(rng.randrange(R))
    pts.append(base[0])
    n = len(ks)
    out = np.zeros((n, 24), dtype=np.uint32)
    assert lib.g_glv_mul(ptr(pack(flat(pts))), ptr(pack(ks)), ptr(out), n) == 0
    v = unpack(out.reshape(-1, 8))
    for j in range(n):
        got = tuple(v[3 * j:3 * j + 3])
        exp = G.mul_scalar(pts[j], ks[j])
        if G.is_zero(exp):
            assert got[2] == 0, (ks[j], pts[j])
        else:
            assert got[2] != 0 and G.affine(got) == G.affine(exp), (ks[j], pts[j])


def test_pairings_plain_fast_and_warp(lib, golden_dir):
    """pairing_affine with the plain and the fast final exponentiation, and the one-warp pairing, on the snarkjs golden
    vk_alfabeta_12, the bn128_test.go literal (e(25 G1, 30 G2) == e(30 G1, 25 G2)) and G1 at infinity."""
    G1, G2 = o.BN.G1, o.BN.G2
    vk = json.load(open(os.path.join(golden_dir, "circom_groth16.json")))["vk"]
    a1 = tuple(int(x) for x in vk["vk_alfa_1"])[:2]
    b2 = tuple(tuple(int(x) for x in c) for c in vk["vk_beta_2"])[:2]
    gold = tuple(tuple(tuple(int(x) for x in f2) for f2 in f6) for f6 in vk["vk_alfabeta_12"])
    p, q = G1.affine(G1.mul_scalar(G1.G, 25)), G2.affine(G2.mul_scalar(G2.G, 30))
    p2, q2 = G1.affine(G1.mul_scalar(G1.G, 30)), G2.affine(G2.mul_scalar(G2.G, 25))
    g1s = [a1, p, p2, (0, 0)]
    g2s = [b2, q[:2], q2[:2], q[:2]]
    n = len(g1s)
    res = []
    for mode in (0, 1, 2):
        out = np.zeros((n, 96), dtype=np.uint32)
        assert lib.g_pairing(mode, ptr(pack(flat(g1s))), ptr(pack(flat(g2s))), ptr(out), n) == 0
        v = unpack(out.reshape(-1, 8))
        res.append([_f12(v[12 * i:12 * (i + 1)]) for i in range(n)])
    e1 = o.BN.pairing((p[0], p[1], 1), (q[0], q[1], (1, 0)))
    assert e1[0][0][0] == 8016119724813186033542830391460394070015218389456422587891475873290878009957   # bn128_test.go:66
    for mode in range(3):
        r = res[mode]
        assert r[0] == gold and r[1] == e1 and r[2] == e1, mode
    assert res[0][3] == res[1][3] == res[2][3]


# ---- the product's element-wise entry points with adversarial operands -------------------------------------------------
@pytest.fixture(scope="module")
def prod():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib


def _limbs(vals):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs(vals)


def _edge_triples(W, n, seed):
    E = arith_edges.edges(Q)
    rng = random.Random(seed)
    el = (lambda: rng.choice(E)) if W == 1 else (lambda: (rng.choice(E), rng.choice(E)))
    return [(el(), el(), el()) for _ in range(n)]


def _group_call(L, name, W, A, B=None, nout=3):
    from gosnark_b200._lib import limbs_to_ints
    n = len(A)
    out = np.zeros((n * nout * W, 4), dtype=np.uint64)
    args = [ptr(_limbs(flat(A)))] + ([ptr(_limbs(flat(B)))] if B is not None else []) + [n, ptr(out)]
    rc = getattr(L, name)(*args)
    return rc, limbs_to_ints(out)


def _check_group_entries(prod, g, A, B):
    G, W = _grp("G1" if g == 1 else "G2")
    L = prod.lib()
    n = len(A)
    for name, fn, nout, two in ((f"b200_g{g}_add_batch", G.add, 3, True), (f"b200_g{g}_double_batch", G.double, 3, False),
                                (f"b200_g{g}_neg_batch", G.neg, 3, False),
                                (f"b200_g{g}_affine_batch", lambda a: _aff(G, a, W), 2, False)):
        rc, got = _group_call(L, name, W, A, B if two else None, nout)
        assert rc == 0, (name, rc)
        exp = [fn(a, b) if two else fn(a) for a, b in zip(A, B)]
        k = nout * W
        bad = [i for i in range(n) if got[k * i:k * (i + 1)] != flat(exp[i])]
        assert not bad, (name, n, len(bad), [(A[i], B[i]) for i in bad[:2]])


@pytest.mark.parametrize("g", [1, 2])
def test_group_entries_edge_triples(prod, g):
    """b200_g{1,2}_{add,double,neg,affine}_batch on arbitrary triples of edge-valued coordinates (2^16 for G1, 2^14 for
    G2), X, Y, Z-exact against the oracle; among them Z = 0 with non-zero X, Y (the other operand comes back), equal
    operands (the reference's Z3 = 0) and curve points with edge-valued Z."""
    W = g
    n = (1 << 16) if g == 1 else (1 << 14)
    A = _edge_triples(W, n, 40 + g)
    B = _edge_triples(W, n, 50 + g)
    G, _ = _grp("G1" if g == 1 else "G2")
    pts = _points("G1" if g == 1 else "G2", 60 + g, 2)
    one = G.F.one()
    zero = G.F.zero()
    nz = A[0][0] if A[0][0] != zero else one
    A[:len(pts)] = pts
    B[:len(pts)] = pts[::-1]
    A[len(pts):2 * len(pts)] = pts                                         # equal operands
    B[len(pts):2 * len(pts)] = pts
    k = 2 * len(pts)
    A[k:k + 4] = [(nz, nz, zero), pts[0], (one, nz, zero), (nz, nz, zero)]  # Z = 0, X, Y != 0 on either side
    B[k:k + 4] = [pts[1], (nz, one, zero), (nz, nz, zero), (one, one, zero)]
    _check_group_entries(prod, g, A, B)


@pytest.mark.parametrize("n", [127, 128, 129])
@pytest.mark.parametrize("g", [1, 2])
def test_group_entries_block_boundaries(prod, g, n):
    """k_group_op / k_group_affine use 128-thread blocks: n just below, at and above one block."""
    _check_group_entries(prod, g, _edge_triples(g, n, n), _edge_triples(g, n, n + 1000))


@pytest.mark.parametrize("g", [1, 2])
def test_group_entries_out_of_range(prod, g):
    """A coordinate equal to q or to 2^256 - 1, in any position of either operand, is B200_ERANGE from every entry; the
    next valid call succeeds."""
    W = g
    L = prod.lib()
    good = _edge_triples(W, 5, 70 + g)
    for bad_val in (Q, (1 << 256) - 1):
        for pos in range(3 * W):
            t = flat(good[2])
            t[pos] = bad_val
            A = list(good)
            A[2] = tuple(t) if W == 1 else tuple((t[2 * j], t[2 * j + 1]) for j in range(3))
            for name, two, nout in ((f"b200_g{g}_add_batch", True, 3), (f"b200_g{g}_double_batch", False, 3),
                                    (f"b200_g{g}_neg_batch", False, 3), (f"b200_g{g}_affine_batch", False, 2)):
                rc, _ = _group_call(L, name, W, A, good if two else None, nout)
                assert rc == -4, (name, bad_val, pos, rc)
                if two:
                    rc, _ = _group_call(L, name, W, good, A, nout)
                    assert rc == -4, (name, "q operand", bad_val, pos, rc)
    _check_group_entries(prod, g, good, good[::-1])


def test_fq12_mul_batch_edge_components(prod):
    """b200_fq12_mul_batch on 2^14 pairs of edge-valued F_q^12 elements against the oracle; a component >= q is
    B200_ERANGE."""
    from gosnark_b200._lib import limbs_to_ints
    L = prod.lib()
    A, B = _f12_elems(1 << 14, 8), _f12_elems(1 << 14, 9)
    n = len(A)
    out = np.zeros((n * 12, 4), dtype=np.uint64)
    assert L.b200_fq12_mul_batch(ptr(_limbs(flat(A))), ptr(_limbs(flat(B))), n, ptr(out)) == 0
    v = limbs_to_ints(out)
    bad = [i for i in range(n) if _f12(v[12 * i:12 * (i + 1)]) != F12.mul(A[i], B[i])]
    assert not bad, (len(bad), [(A[i], B[i]) for i in bad[:1]])
    for bad_val in (Q, (1 << 256) - 1):
        x = flat(A[:2])
        x[17] = bad_val
        assert L.b200_fq12_mul_batch(ptr(_limbs(x)), ptr(_limbs(flat(B[:2]))), 2, ptr(out)) == -4
        assert L.b200_fq12_mul_batch(ptr(_limbs(flat(B[:2]))), ptr(_limbs(x)), 2, ptr(out)) == -4
    assert L.b200_fq12_mul_batch(ptr(_limbs(flat(A[:2]))), ptr(_limbs(flat(B[:2]))), 2, ptr(out)) == 0


@pytest.mark.parametrize("g", [1, 2])
def test_mul_batch_edge_points_and_scalars(prod, g):
    """b200_g{1,2}_mul_batch (the reference's MSB-first double-and-add) X, Y, Z-exactly on curve points with edge-valued
    Z and on edge-coordinate triples, times edge scalars (0, 1, 2, r - 1, r, 2^128 +- 1, 2^255, 2^256 - 1); a coordinate
    >= q is B200_ERANGE."""
    from gosnark_b200._lib import limbs_to_ints
    G, W = _grp("G1" if g == 1 else "G2")
    L = prod.lib()
    scal = [0, 1, 2, 3, R - 1, R, (1 << 128) - 1, (1 << 128) + 1, 1 << 255, (1 << 256) - 1]
    pts = _points("G1" if g == 1 else "G2", 80 + g, 1) + _edge_triples(W, 4, 90 + g)
    rng = random.Random(g)
    cases = [(pts[i % len(pts)], s) for i, s in enumerate(scal)] + [(rng.choice(pts), rng.choice(scal)) for _ in range(14)]
    n = len(cases)
    out = np.zeros((n * 3 * W, 4), dtype=np.uint64)
    name = f"b200_g{g}_mul_batch"
    assert getattr(L, name)(ptr(_limbs(flat([c[0] for c in cases]))), ptr(_limbs([c[1] for c in cases])), n, ptr(out)) == 0
    v = limbs_to_ints(out)
    for i, (P, s) in enumerate(cases):
        assert v[3 * W * i:3 * W * (i + 1)] == flat(G.mul_scalar(P, s)), (P, s)
    bad = flat(pts[:1])
    bad[0] = Q
    assert getattr(L, name)(ptr(_limbs(bad)), ptr(_limbs([5])), 1, ptr(out)) == -4
