"""CPU unit tests of the kernel arithmetic headers (fp.cuh / fp2.cuh / ec.cuh)
compiled for the host through the carry-flag emulation in hd.cuh, checked
against the oracle.  Exercises the chain logic the device code runs, on the
edge vectors of tests/arith_edges.py; no GPU needed.  tests/test_gpu_arith.py
(-m gpu) runs the same vectors through the same headers compiled by nvcc for
sm_90a, in both the inlined and the outlined build variants."""
import ctypes
import os
import random

import numpy as np
import pytest

import arith_edges
import build as b200build
from oracle import ref_py as o

Q, R = o.Q, o.R


@pytest.fixture(scope="module")
def lib():
    path = b200build.build_host_arith()
    return ctypes.CDLL(path)


def to_u32(vals):
    """list of ints -> uint32 array, 8 limbs each, little endian."""
    buf = b"".join(int(v).to_bytes(32, "little") for v in vals)
    return np.frombuffer(buf, dtype=np.uint32).copy()


def from_u32(arr, n):
    raw = arr.tobytes()
    return [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(n)]


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def call(fn, *args, nout):
    out = np.zeros(8 * nout, dtype=np.uint32)
    fn(*args, ptr(out))
    return from_u32(out, nout)


def call_canon(fn, *args, nout):
    """call() of t_fp_op / t_fq2_op that also requires the Montgomery result to be canonical (< p): the conversion out
    of Montgomery form reduces, so a missing final subtraction shows only in this flag."""
    out = np.zeros(8 * nout, dtype=np.uint32)
    assert fn(*args, ptr(out)) == 0, "Montgomery result >= p"
    return from_u32(out, nout)


EDGE = [0, 1, 2, 3]


def samples(p, rng, k=200):
    vals = EDGE + [p - 1, p - 2, (p - 1) // 2, (1 << 253) % p, (1 << 128), (1 << 32) - 1, (1 << 224) - 1]
    vals += [rng.randrange(p) for _ in range(k)]
    return vals


@pytest.mark.parametrize("field,p", [(0, Q), (1, R)], ids=["Fq", "Fr"])
def test_fp_edge_pairs(lib, field, p):
    """Every pair of the shared edge set (standard-form edges and their Montgomery preimages) through add, sub and mul,
    every edge through neg, sqr and both inversions, and geq_modulus at either side of p."""
    E = arith_edges.edges(p)
    bufs = [to_u32([v]) for v in E]
    for a, A in zip(E, bufs):
        for b, B in zip(E, bufs):
            assert call_canon(lib.t_fp_op, field, 0, ptr(A), ptr(B), nout=1)[0] == (a + b) % p, (hex(a), hex(b))
            assert call_canon(lib.t_fp_op, field, 1, ptr(A), ptr(B), nout=1)[0] == (a - b) % p, (hex(a), hex(b))
            assert call_canon(lib.t_fp_op, field, 2, ptr(A), ptr(B), nout=1)[0] == a * b % p, (hex(a), hex(b))
        assert call_canon(lib.t_fp_op, field, 4, ptr(A), ptr(A), nout=1)[0] == (-a) % p, hex(a)
        assert call_canon(lib.t_fp_op, field, 5, ptr(A), ptr(A), nout=1)[0] == a * a % p, hex(a)
        inv = pow(a, -1, p) if a else 0
        assert call_canon(lib.t_fp_op, field, 3, ptr(A), ptr(A), nout=1)[0] == inv, hex(a)
        assert call_canon(lib.t_fp_op, field, 6, ptr(A), ptr(A), nout=1)[0] == inv, hex(a)
        assert lib.t_geq(field, ptr(A)) == 0, hex(a)
    for v in (p, p + 1, p + (1 << 32), (1 << 256) - 1, (1 << 255), p | 0xffffffff):
        assert lib.t_geq(field, ptr(to_u32([v]))) == 1, hex(v)


@pytest.mark.parametrize("field,p", [(0, Q), (1, R)])
def test_fp_ops(lib, field, p):
    rng = random.Random(1234 + field)
    vs = samples(p, rng)
    for i, a in enumerate(vs):
        b = vs[(i * 7 + 3) % len(vs)]
        A, B = to_u32([a]), to_u32([b])
        assert call_canon(lib.t_fp_op, field, 0, ptr(A), ptr(B), nout=1)[0] == (a + b) % p
        assert call_canon(lib.t_fp_op, field, 1, ptr(A), ptr(B), nout=1)[0] == (a - b) % p
        assert call_canon(lib.t_fp_op, field, 2, ptr(A), ptr(B), nout=1)[0] == (a * b) % p
        assert call_canon(lib.t_fp_op, field, 4, ptr(A), ptr(B), nout=1)[0] == (-a) % p
    for a in vs[:40]:
        A = to_u32([a])
        exp = pow(a, -1, p) if a else 0
        assert call_canon(lib.t_fp_op, field, 3, ptr(A), ptr(A), nout=1)[0] == exp
    for a in vs + [1 << k for k in range(0, 254, 7)] + [p - (1 << k) for k in range(1, 250, 11)]:
        A = to_u32([a])                               # binary-Euclid inversion: same value as a^(p-2)
        exp = pow(a, -1, p) if a else 0
        assert call_canon(lib.t_fp_op, field, 6, ptr(A), ptr(A), nout=1)[0] == exp
    assert lib.t_geq(field, ptr(to_u32([p]))) == 1
    assert lib.t_geq(field, ptr(to_u32([p - 1]))) == 0
    assert lib.t_geq(field, ptr(to_u32([(1 << 256) - 1]))) == 1


def test_wide_product_and_reduction(lib):
    """mul_full == the integer product for arbitrary 256-bit operands (carries at every limb boundary) and
    redc_wide == t / 2^256 mod p: the two halves of the lazily reduced F_q^2 multiply."""
    rng = random.Random(2024)
    M = (1 << 256) - 1
    H = (1 << 128) - 1
    edge = [0, 1, M, H, H << 128, (1 << 128), (1 << 255), M - 1, (H << 128) | 1, 0xffffffff, 0xffffffff << 96,
            sum(0xffffffff << (64 * i) for i in range(4)), sum(0xffffffff << (64 * i + 32) for i in range(4))]
    vals = edge + [rng.randrange(1 << 256) for _ in range(150)] + [rng.randrange(1 << 128) for _ in range(10)]
    for i, a in enumerate(vals):
        for b in (vals[(i * 7 + 3) % len(vals)], vals[(i * 13 + 5) % len(edge)], a):
            A, B = to_u32([a]), to_u32([b])
            for k in (0,):
                out = np.zeros(16, dtype=np.uint32)
                lib.t_mul_full(k, ptr(A), ptr(B), ptr(out))
                assert int.from_bytes(out.tobytes(), "little") == a * b, (k, hex(a), hex(b))
    for field, p in ((0, Q), (1, R)):
        # wide reduction t -> t / 2^256 mod p for t < p * 2^256 (extremes: 0, p*2^256 - 1, all-ones low half)
        rinv = pow(1 << 256, -1, p)
        ts = [0, 1, p * (1 << 256) - 1, (1 << 256) - 1, (p - 1) * (p - 1), ((1 << 256) - 1) * (p - 1), p << 255] + \
             [rng.randrange(p << 256) for _ in range(200)]
        for t in ts:
            T = np.frombuffer(int(t).to_bytes(64, "little"), dtype=np.uint32).copy()
            for k in (0,):
                out = np.zeros(8, dtype=np.uint32)
                lib.t_redc_wide(field, k, ptr(T), ptr(out))
                assert int.from_bytes(out.tobytes(), "little") == (t * rinv) % p, (field, k, hex(t))


def test_fq2_ops(lib):
    rng = random.Random(99)
    F2 = o.BN.Fq2
    vs = samples(Q, rng, 60)
    for i in range(len(vs)):
        a = (vs[i], vs[(i * 5 + 1) % len(vs)])
        b = (vs[(i * 3 + 2) % len(vs)], vs[(i * 11 + 7) % len(vs)])
        A, B = to_u32(a), to_u32(b)
        assert tuple(call(lib.t_fq2_op, 0, ptr(A), ptr(B), nout=2)) == F2.add(a, b)
        assert tuple(call(lib.t_fq2_op, 1, ptr(A), ptr(B), nout=2)) == F2.sub(a, b)
        assert tuple(call(lib.t_fq2_op, 2, ptr(A), ptr(B), nout=2)) == F2.mul(a, b)      # fq2.go:63-76
        assert tuple(call(lib.t_fq2_op, 4, ptr(A), ptr(B), nout=2)) == F2.square(a)      # fq2.go:118-133
        assert tuple(call(lib.t_fq2_op, 5, ptr(A), ptr(B), nout=2)) == F2.neg(a)
        if a != (0, 0) and i < 25:
            assert tuple(call(lib.t_fq2_op, 3, ptr(A), ptr(B), nout=2)) == F2.inverse(a)  # fq2.go:99-108
            assert tuple(call(lib.t_fq2_op, 6, ptr(A), ptr(B), nout=2)) == F2.inverse(a)


def test_wide_edges(lib):
    """mul_full on every pair of the shared wide edges (up to (2^256 - 1)^2) and redc_wide on the shared reduction edges
    (up to t = p * 2^256 - 1), for both moduli."""
    W = arith_edges.wide_edges()
    for a in W:
        for b in W:
            out = np.zeros(16, dtype=np.uint32)
            lib.t_mul_full(0, ptr(to_u32([a])), ptr(to_u32([b])), ptr(out))
            assert int.from_bytes(out.tobytes(), "little") == a * b, (hex(a), hex(b))
    for field, p in ((0, Q), (1, R)):
        rinv = pow(1 << 256, -1, p)
        for t in arith_edges.redc_edges(p):
            out = np.zeros(8, dtype=np.uint32)
            lib.t_redc_wide(field, 0, ptr(np.frombuffer(t.to_bytes(64, "little"), dtype=np.uint32).copy()), ptr(out))
            assert int.from_bytes(out.tobytes(), "little") == t * rinv % p, (field, hex(t))


def test_fq2_edge_components(lib):
    """F_q^2 products, squares, sums and differences with components drawn from the shared edge set, including the
    lazy-reduction extremes in Montgomery form: a0 b0 = 0 with a1 b1 maximal (the representatives p - 1) and the reverse."""
    F2 = o.BN.Fq2
    E = arith_edges.edges(Q)
    m1 = arith_edges.montgomery_preimages(Q, [Q - 1])[0]       # Montgomery representative p - 1
    pairs = [((0, m1), (x, m1)) for x in E] + [((m1, 0), (m1, x)) for x in E]
    rng = random.Random(5)
    pairs += [((rng.choice(E), rng.choice(E)), (rng.choice(E), rng.choice(E))) for _ in range(1500)]
    for a, b in pairs:
        A, B = to_u32(a), to_u32(b)
        assert tuple(call_canon(lib.t_fq2_op, 2, ptr(A), ptr(B), nout=2)) == F2.mul(a, b), (a, b)
        assert tuple(call_canon(lib.t_fq2_op, 0, ptr(A), ptr(B), nout=2)) == F2.add(a, b), (a, b)
        assert tuple(call_canon(lib.t_fq2_op, 1, ptr(A), ptr(B), nout=2)) == F2.sub(a, b), (a, b)
        assert tuple(call_canon(lib.t_fq2_op, 4, ptr(A), ptr(B), nout=2)) == F2.square(a), a


def test_fq2_lazy_reduction_extremes(lib):
    """The lazily reduced product keeps 512-bit intermediates: exercise the bound cases
    (all components p-1, zero, v0 < v1, v0 > v1)."""
    F2 = o.BN.Fq2
    ext = [0, 1, Q - 1, Q - 2, (Q - 1) // 2, 2]
    for a0 in ext:
        for a1 in ext:
            for b0, b1 in ((Q - 1, Q - 1), (0, Q - 1), (Q - 1, 0), (1, 1), (Q - 2, 3)):
                a, b = (a0, a1), (b0, b1)
                assert tuple(call(lib.t_fq2_op, 2, ptr(to_u32(a)), ptr(to_u32(b)), nout=2)) == F2.mul(a, b)


def _flat(pt):
    out = []
    for c in pt:
        out.extend(c if isinstance(c, tuple) else (c,))
    return out


def _xyzz_of(group, jac, F):
    """Jacobian -> XYZZ (X, Y, Z^2, Z^3)."""
    zz = F.square(jac[2])
    return (jac[0], jac[1], zz, F.mul(zz, jac[2]))


@pytest.mark.parametrize("gname", ["G1", "G2"])
def test_xyzz_group_law(lib, gname):
    grp = getattr(o.BN, gname)
    F = grp.F
    W = 1 if gname == "G1" else 2
    fn = lib.t_g1_xyzz if gname == "G1" else lib.t_g2_xyzz
    zero_aff = (0, 0) if W == 1 else ((0, 0), (0, 0))
    rng = random.Random(7)

    def aff(p):                      # oracle affine -> ((x),(y)) with our (0,0) infinity convention
        if grp.is_zero(p):
            return zero_aff
        a = grp.affine(p)
        return (a[0], a[1])

    ks = [rng.randrange(1, R) for _ in range(6)]
    pts = [grp.mul_scalar(grp.G, k) for k in ks]     # Jacobian with Z != 1
    inf = grp.zero3()
    for i, P in enumerate(pts):
        Qp = pts[(i + 1) % len(pts)]
        PX = to_u32(_flat(_xyzz_of(grp, P, F)))
        # madd with affine Q
        qa = aff(Qp)
        out = call(fn, 0, ptr(PX), ptr(to_u32(_flat(qa))), nout=2 * W)
        assert out == _flat(aff(grp.add(P, Qp)))
        # general add
        out = call(fn, 1, ptr(PX), ptr(to_u32(_flat(_xyzz_of(grp, Qp, F)))), nout=2 * W)
        assert out == _flat(aff(grp.add(P, Qp)))
        # doubling
        out = call(fn, 2, ptr(PX), ptr(PX), nout=2 * W)
        assert out == _flat(aff(grp.double(P)))
        # xyzz <-> jacobian round trip keeps the point
        out = call(fn, 3, ptr(PX), ptr(PX), nout=2 * W)
        assert out == _flat(aff(P))
        # P + P through madd / add must double (reference Add would return infinity, H6)
        out = call(fn, 0, ptr(PX), ptr(to_u32(_flat(aff(P)))), nout=2 * W)
        assert out == _flat(aff(grp.double(P)))
        out = call(fn, 1, ptr(PX), ptr(PX), nout=2 * W)
        assert out == _flat(aff(grp.double(P)))
        # P + (-P) = infinity
        out = call(fn, 0, ptr(PX), ptr(to_u32(_flat(aff(grp.neg(P))))), nout=2 * W)
        assert out == _flat(zero_aff)
        out = call(fn, 1, ptr(PX), ptr(to_u32(_flat(_xyzz_of(grp, grp.neg(P), F)))), nout=2 * W)
        assert out == _flat(zero_aff)
        # infinity handling both sides
        IX = to_u32(_flat(_xyzz_of(grp, inf, F)))
        out = call(fn, 0, ptr(IX), ptr(to_u32(_flat(aff(P)))), nout=2 * W)
        assert out == _flat(aff(P))
        out = call(fn, 0, ptr(PX), ptr(to_u32(_flat(zero_aff))), nout=2 * W)
        assert out == _flat(aff(P))
        out = call(fn, 1, ptr(IX), ptr(PX), nout=2 * W)
        assert out == _flat(aff(P))
        out = call(fn, 1, ptr(PX), ptr(IX), nout=2 * W)
        assert out == _flat(aff(P))


@pytest.mark.parametrize("gname", ["G1", "G2"])
def test_reference_formulas_exact_jacobian(lib, gname):
    """jac_add_ref / jac_double_ref reproduce g1.go:32-138 / g2.go:32-140 X,Y,Z-exactly."""
    grp = getattr(o.BN, gname)
    W = 1 if gname == "G1" else 2
    fn = lib.t_g1_jac if gname == "G1" else lib.t_g2_jac
    rng = random.Random(11)
    pts = [grp.mul_scalar(grp.G, rng.randrange(1, R)) for _ in range(4)] + [grp.G]
    for i, P in enumerate(pts):
        Qp = pts[(i + 1) % len(pts)]
        A, B = to_u32(_flat(P)), to_u32(_flat(Qp))
        assert call(fn, 0, ptr(A), ptr(B), nout=3 * W) == _flat(grp.add(P, Qp))
        assert call(fn, 1, ptr(A), ptr(B), nout=3 * W) == _flat(grp.double(P))
