"""CPU: the batched Groth16 verifier's kernels (csrc/verify_batch.cuh) and the pairing split they rely on, over emulated
CTAs (tests/host/verify_batch_test.cpp, csrc/host_stub), against the oracle.

- The split pairings: wp::miller_loop then wp::final_exp (in separate launches) equals wp::pairing, pairing_affine_t and
  miller_loop_affine + final_exp_fast word for word, and the oracle's bn128.Pairing.
- FE(ML_1 * ML_2) through k_vb_product equals e_1 * e_2; k_vb_final's aggregate bit says whether it is one.
- The G2 subgroup test (psi(Q) == [6u^2]Q) equals [r]Q == O on the oracle, on multiples of the generator and on twist
  points off the subgroup built by an F_q^2 square root on random x (and on their [r] multiples).
- k_vb_classify: infinity, off-curve and off-subgroup inputs, coordinates >= q, an irregular Vk.
- The aggregate on small batches with fixed rho, kernel by kernel in the library's order: valid batches pass, one bad
  proof fails it, two bad proofs that cancel under rho = (1, 1) pass only there, irregular proofs stay out of it."""
import ctypes
import random

import numpy as np
import pytest

import build as b200build
from oracle import ref_py as o

G1, G2 = o.BN.G1, o.BN.G2
R, Q = o.R, o.Q
F2 = o.BN.Fq2
TB = o.BN.twist_coef_b


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_verify_batch())


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def u64(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint64).copy()


def g1w(p):
    return [p[0], p[1], p[2]]


def g2w(p):
    return [p[0][0], p[0][1], p[1][0], p[1][1], p[2][0], p[2][1]]


def f12_of(out):
    raw = out.tobytes()
    v = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(12)]
    return tuple(tuple((v[6 * h + 2 * k], v[6 * h + 2 * k + 1]) for k in range(3)) for h in range(2))


def aff_g1(p):
    x, y = G1.affine(p)[:2]
    return u32([x, y])


def aff_g2(p):
    a = G2.affine(p)
    return u32([a[0][0], a[0][1], a[1][0], a[1][1]])


# ---- F_q^2 square roots and twist points off the subgroup ----------------------------------------------------------
def fq_sqrt(a):
    s = pow(a, (Q + 1) // 4, Q)
    return s if s * s % Q == a % Q else None


def fq2_sqrt(a):
    a0, a1 = a
    t = fq_sqrt((a0 * a0 + a1 * a1) % Q)
    if t is None:
        return None
    inv2 = pow(2, -1, Q)
    for tt in (t, Q - t):
        x0 = fq_sqrt((a0 + tt) * inv2 % Q)
        if x0:
            x1 = a1 * pow(2 * x0, -1, Q) % Q
            if F2.square((x0, x1)) == (a0 % Q, a1 % Q):
                return (x0, x1)
    return None


def twist_point(rng):
    """(x, y, 1) on y^2 = x^3 + b' for a random x: of order r times a cofactor part, almost never in G2."""
    while True:
        x = (rng.randrange(Q), rng.randrange(Q))
        y = fq2_sqrt(F2.add(F2.mul(F2.square(x), x), TB))
        if y is not None:
            return (x, y, (1, 0))


def in_subgroup_oracle(p):
    return G2.is_zero(G2.mul_scalar(p, R))


# ---- the split pairings ----------------------------------------------------------------------------------------------
def test_pairing_split_word_for_word(lib):
    rng = random.Random(7)
    for trial in range(2):
        p = G1.mul_scalar(G1.G, rng.randrange(1, R))
        q = G2.mul_scalar(G2.G, rng.randrange(1, R))
        out = np.zeros(96, np.uint32)
        assert lib.t_vb_pairing_split(_p(aff_g1(p)), _p(aff_g2(q)), _p(out)) == 0
        if trial == 0:
            assert f12_of(out) == o.BN.pairing(p, q)


def test_fe_of_miller_product_is_product_of_pairings(lib):
    rng = random.Random(8)
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    p1, q1 = G1.mul_scalar(G1.G, a), G2.mul_scalar(G2.G, b)
    out = np.zeros(96, np.uint32)
    # two unrelated pairs: the value is e_1 * e_2 != 1
    p2, q2 = G1.mul_scalar(G1.G, rng.randrange(1, R)), G2.mul_scalar(G2.G, rng.randrange(1, R))
    assert lib.t_vb_fe_of_product(_p(aff_g1(p1)), _p(aff_g2(q1)), _p(aff_g1(p2)), _p(aff_g2(q2)), _p(out)) == 0
    # e(aP, bQ) * e(-abP, Q) = 1: the aggregate bit must be set
    p3 = G1.neg(G1.mul_scalar(G1.G, a * b % R))
    assert lib.t_vb_fe_of_product(_p(aff_g1(p1)), _p(aff_g2(q1)), _p(aff_g1(p3)), _p(aff_g2(G2.G)), _p(out)) == 0
    assert f12_of(out) == o.BN.Fq12.one()


# ---- G2 subgroup test ------------------------------------------------------------------------------------------------
def test_g2_subgroup_matches_r_times_q(lib):
    rng = random.Random(9)
    h = 2 * Q - R                                     # the twist's cofactor
    pts = [G2.G, G2.mul_scalar(G2.G, R - 1), G2.mul_scalar(G2.G, rng.randrange(1, R))]
    off = [twist_point(rng) for _ in range(4)]
    pts += off
    pts += [G2.mul_scalar(off[0], R)]                 # order divides the cofactor: off the subgroup
    pts += [G2.mul_scalar(off[1], h)]                 # cleared cofactor: in the subgroup
    pts += [G2.double(off[2])]
    want = [1 if in_subgroup_oracle(p) else 0 for p in pts]
    assert want[:3] == [1, 1, 1] and want[3:7] == [0, 0, 0, 0] and want[7] == 0 and want[8] == 1
    got = np.zeros(len(pts), np.int32)
    words = u32([w for p in pts for w in g2w(p)])
    assert lib.t_vb_g2_subgroup(_p(words), len(pts), _p(got)) == 0
    assert list(got) == want


# ---- proofs with known discrete logs ---------------------------------------------------------------------------------
class Key:
    """A Vk with known discrete logs: alpha1 = a G1, beta2 = b G2, gamma2 = g G2, delta2 = d G2, IC_j = ic_j G1."""

    def __init__(self, npub, seed):
        rng = random.Random(seed)
        self.a, self.b, self.g, self.d = (rng.randrange(1, R) for _ in range(4))
        self.ic = [rng.randrange(1, R) for _ in range(npub + 1)]
        self.npub = npub
        self.alpha = G1.mul_scalar(G1.G, self.a)
        self.beta, self.gamma, self.delta = (G2.mul_scalar(G2.G, k) for k in (self.b, self.g, self.d))
        self.IC = [G1.mul_scalar(G1.G, k) for k in self.ic]

    def vk_words(self):
        return u64(g1w(self.alpha) + g2w(self.beta) + g2w(self.gamma) + g2w(self.delta))

    def ic_words(self):
        return u64([w for p in self.IC for w in g1w(p)])

    def proof(self, pub, x, y):
        """A = x G1, B = y G2, C = c G1 with x y = a b + I g + c d, I = ic_0 + sum pub_j ic_{j+1}."""
        i = (self.ic[0] + sum(s * k for s, k in zip(pub, self.ic[1:]))) % R
        c = (x * y - self.a * self.b - i * self.g) * pow(self.d, -1, R) % R
        return [G1.mul_scalar(G1.G, x), G2.mul_scalar(G2.G, y), G1.mul_scalar(G1.G, c)]


def proof_words(proofs):
    return u64([w for a, b, c in proofs for w in g1w(a) + g1w(c) + g2w(b)])


def aggregate(lib, key, proofs, pubs, rho, warp=False):
    k = len(proofs)
    flags = np.zeros(k + 1, np.uint32)
    icp = np.zeros(12 * k, np.uint64)
    agg, status = ctypes.c_uint32(0), ctypes.c_uint32(0)
    pub = u64([s for ps in pubs for s in ps]) if key.npub else np.zeros(4, np.uint64)
    rl = np.array([w for r in rho for w in (r & (2**64 - 1), r >> 64)], dtype=np.uint64)
    k_reg = lib.t_vb_aggregate(_p(key.ic_words()), _p(key.vk_words()), _p(proof_words(proofs)), _p(pub), key.npub, k, _p(rl),
                               int(warp), _p(flags), _p(icp), ctypes.byref(agg), ctypes.byref(status))
    return k_reg, agg.value, status.value, list(flags)


@pytest.fixture(scope="module")
def batch():
    key = Key(2, 11)
    rng = random.Random(12)
    pubs = [[rng.randrange(R) for _ in range(2)] for _ in range(3)]
    proofs = [key.proof(ps, rng.randrange(1, R), rng.randrange(1, R)) for ps in pubs]
    return key, proofs, pubs


RHO = [0x1234567890abcdef1122334455667788, 0xfedcba0987654321a1b2c3d4e5f60718, 3]


def test_aggregate_valid_batch_passes(lib, batch):
    key, proofs, pubs = batch
    k_reg, agg, status, flags = aggregate(lib, key, proofs, pubs, RHO)
    assert (k_reg, agg, status, flags) == (3, 1, 1, [0, 0, 0, 0])


def test_aggregate_valid_batch_warp_miller(lib, batch):
    key, proofs, pubs = batch
    assert aggregate(lib, key, proofs[:1], pubs[:1], RHO[:1], warp=True)[:3] == (1, 1, 1)


def test_aggregate_icpubl_matches_oracle_sum(lib, batch):
    """icPubl_i is the reference's sum (oracle add, reference order), as a group element."""
    key, proofs, pubs = batch
    flags = np.zeros(4, np.uint32)
    icp = np.zeros(36, np.uint64)
    agg, status = ctypes.c_uint32(0), ctypes.c_uint32(0)
    rl = np.array([w for r in RHO for w in (r & (2**64 - 1), r >> 64)], dtype=np.uint64)
    lib.t_vb_aggregate(_p(key.ic_words()), _p(key.vk_words()), _p(proof_words(proofs)), _p(u64([s for ps in pubs for s in ps])),
                       2, 3, _p(rl), 0, _p(flags), _p(icp), ctypes.byref(agg), ctypes.byref(status))
    raw = icp.tobytes()
    for i, ps in enumerate(pubs):
        got = tuple(int.from_bytes(raw[96 * i + 32 * j:96 * i + 32 * j + 32], "little") for j in range(3))
        want = key.IC[0]
        for s, p in zip(ps, key.IC[1:]):
            want = G1.add(want, G1.mul_scalar(p, s))
        assert G1.affine(got) == G1.affine(want)


def test_aggregate_one_bad_proof_fails(lib, batch):
    key, proofs, pubs = batch
    bad = [list(p) for p in proofs]
    bad[1][2] = G1.add(bad[1][2], G1.G)                # C + G
    assert aggregate(lib, key, bad, pubs, RHO)[:3] == (3, 0, 0)


def test_aggregate_cancelling_pair_needs_random_rho(lib, batch):
    key, proofs, pubs = batch
    d = G1.mul_scalar(G1.G, 0xC0FFEE)
    bad = [list(p) for p in proofs]
    bad[0][2] = G1.add(bad[0][2], d)
    bad[2][2] = G1.add(bad[2][2], G1.neg(d))
    assert aggregate(lib, key, bad, pubs, [1, 1, 1])[:3] == (3, 1, 1)
    assert aggregate(lib, key, bad, pubs, RHO)[:3] == (3, 0, 0)


def test_classification_and_irregular_proofs_stay_out(lib, batch):
    key, proofs, pubs = batch
    rng = random.Random(13)
    cases = {
        "A at infinity": lambda p: [(0, 0, 0), p[1], p[2]],
        "C at infinity": lambda p: [p[0], p[1], (1, 1, 0)],
        "A off the curve": lambda p: [(p[0][0], (p[0][1] + 1) % Q, p[0][2]), p[1], p[2]],
        "B off the subgroup": lambda p: [p[0], twist_point(rng), p[2]],
    }
    for name, mk in cases.items():
        bad = [list(p) for p in proofs]
        bad[1] = mk(bad[1])
        k_reg, agg, status, flags = aggregate(lib, key, bad, pubs, RHO)
        assert flags == [0, 1, 0, 0], name
        assert (k_reg, agg, status) == (2, 1, 1 | 4), name
    # PiB at infinity and a coordinate >= q: bad (verdict 0 without a pairing); the Vk off its subgroup: nothing aggregated
    vk = key.vk_words()
    flags = np.zeros(4, np.uint32)
    st = ctypes.c_uint32(0)
    bad = [list(p) for p in proofs]
    bad[0][1] = ((1, 0), (1, 0), (0, 0))
    bad[2][0] = (Q, 1, 1)
    assert lib.t_vb_classify(_p(proof_words(bad)), _p(vk), 3, _p(flags), ctypes.byref(st)) == 0
    assert list(flags) == [3, 0, 3, 0] and st.value == 4 | 8
    key2 = Key(2, 11)
    key2.beta = twist_point(rng)
    assert lib.t_vb_classify(_p(proof_words(proofs)), _p(key2.vk_words()), 3, _p(flags), ctypes.byref(st)) == 0
    assert list(flags) == [0, 0, 0, 1] and st.value == 4
    assert aggregate(lib, key2, proofs, pubs, RHO)[:3] == (0, 0, 4)


def test_icpubl_at_infinity_is_irregular(lib):
    """IC[0] + s IC[1] = O for s = -ic_0 / ic_1: the proof pairs (0, 0) in the reference, so it stays out."""
    key = Key(1, 21)
    s = (-key.ic[0]) * pow(key.ic[1], -1, R) % R
    rng = random.Random(22)
    pubs = [[s], [rng.randrange(R)]]
    proofs = [key.proof(ps, rng.randrange(1, R), rng.randrange(1, R)) for ps in pubs]
    k_reg, agg, status, flags = aggregate(lib, key, proofs, pubs, RHO[:2])
    assert flags == [1, 0, 0] and (k_reg, agg, status) == (1, 1, 1 | 4)
