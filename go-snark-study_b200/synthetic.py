"""Synthetic Groth16 workloads with KNOWN DISCRETE LOGS (SURVEY §8c/§8d).

Shape: n constraints, m = n + 2 signals, NPublic = 1 (the only shape the
reference supports, SURVEY H5).  Every CRS point is k*G for a seeded k, minted on
the GPU with the reference-order batch MulScalar, so the exact proof the
reference's GenerateProofs would return on the same (pk, w, px, r, s) is known
in the exponent and costs one CPU scalar multiplication per proof element to
check — bit-exact parity at 2^16 / 2^20 without an O(n) CPU run.

px is minted as h0 * Z (GPU product) for a seeded h0 and a seeded monic Z of
degree n, so the division is exact and h must come back equal to h0.
"""
import numpy as np

from . import _lib
from ._lib import check, ints_to_limbs, lib, limbs_to_ints, ptr
from .bn128 import G1, G2, R, _flatten_g1, _flatten_g2

SEED_WITNESS, SEED_TOXIC, SEED_RS, SEED_POINTS, SEED_SCALARS = 0x5EED0001, 0x5EED0002, 0x5EED0003, 0x5EED0004, 0x5EED0005


def rand_limbs(n, seed):
    """n scalars uniform in [0, 2^253) (< r), as (n, 4) uint64 limbs."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 61) - 1)
    return np.ascontiguousarray(a)


def mint_points(group, dlog_limbs):
    """[k_i * G] as Jacobian standard-form limbs, via b200_g*_mul_batch_bcast."""
    n = dlog_limbs.shape[0]
    words = 12 if group == 1 else 24
    gen = _flatten_g1([G1.G]) if group == 1 else _flatten_g2([G2.G])
    out = np.zeros((n, words), dtype=np.uint64)
    fn = lib().b200_g1_mul_batch_bcast if group == 1 else lib().b200_g2_mul_batch_bcast
    check(fn(ptr(gen), ptr(dlog_limbs), n, ptr(out)))
    return out


class SyntheticGroth16:
    def __init__(self, logn, mint=True):
        self.logn = logn
        n = self.n = 1 << logn
        m = self.m = n + 2
        self.npublic = 1
        self.n_ptd = m - 1
        # discrete logs of the CRS arrays
        self.k_at = rand_limbs(m, SEED_POINTS)
        self.k_b = rand_limbs(m, SEED_POINTS + 1)
        self.k_c = rand_limbs(m, SEED_POINTS + 2)
        self.k_c[: self.npublic + 1] = 0                      # BACDelta[0..NPublic] = (0,0,0), groth16.go:177-180
        self.k_ptd = rand_limbs(self.n_ptd, SEED_POINTS + 3)
        tox = rand_limbs(3, SEED_TOXIC)
        self.k_alpha, self.k_beta, self.k_delta = (tox[i:i + 1] for i in range(3))
        self.w = rand_limbs(m, SEED_WITNESS)
        self.w[0] = (1, 0, 0, 0)                              # signal "one"
        rs = limbs_to_ints(rand_limbs(2, SEED_RS))
        self.r, self.s = rs[0] >> 13, rs[1] >> 13             # 240-bit, the range of Fq.Rand (H2)
        self.h0 = rand_limbs(n - 1, SEED_SCALARS)
        self.z = rand_limbs(n + 1, SEED_SCALARS + 1)
        self.z[n] = (1, 0, 0, 0)                              # monic, degree n = m - 2 (groth16.go:122-132)
        if mint:
            self.mint()

    def mint(self):
        self.at = mint_points(1, self.k_at)
        self.b1 = mint_points(1, self.k_b)
        self.b2 = mint_points(2, self.k_b)
        self.cd = mint_points(1, self.k_c)
        self.ptd = mint_points(1, self.k_ptd)
        self.alpha1, self.beta1, self.delta1 = (mint_points(1, k) for k in (self.k_alpha, self.k_beta, self.k_delta))
        self.beta2, self.delta2 = (mint_points(2, k) for k in (self.k_beta, self.k_delta))
        n = self.n
        self.px = np.zeros((2 * n - 1, 4), dtype=np.uint64)
        check(lib().b200_poly_mul(ptr(self.h0), n - 1, ptr(self.z), n + 1, ptr(self.px)))

    def load_pk(self, rank=0, world=1, window_bits=0):
        h = _lib._h(0)
        check(lib().b200_groth16_pk_load_shard(
            ptr(self.at), ptr(self.b1), ptr(self.b2), ptr(self.cd), self.m, ptr(self.ptd), self.n_ptd,
            ptr(self.z), self.z.shape[0], ptr(self.alpha1), ptr(self.beta1), ptr(self.delta1), ptr(self.beta2),
            ptr(self.delta2), self.npublic, window_bits, rank, world, h))
        return h.value

    def pk_dict(self):
        """The same key as a groth16.Pk-shaped dict of Python ints (small sizes only)."""
        from .bn128 import _unflatten_g1, _unflatten_g2
        return {"Z": limbs_to_ints(self.z), "BACDelta": _unflatten_g1(self.cd), "PowersTauDelta": _unflatten_g1(self.ptd),
                "G1": {"Alpha": _unflatten_g1(self.alpha1)[0], "Beta": _unflatten_g1(self.beta1)[0],
                       "Delta": _unflatten_g1(self.delta1)[0], "At": _unflatten_g1(self.at),
                       "BACGamma": _unflatten_g1(self.b1)},
                "G2": {"Beta": _unflatten_g2(self.beta2)[0], "Delta": _unflatten_g2(self.delta2)[0],
                       "BACGamma": _unflatten_g2(self.b2)}}

    def expected_dlogs(self, r=None, s=None):
        """Discrete logs (w.r.t. the generators) of PiA, PiB, PiC that
        groth16.GenerateProofs (groth16.go:225-278) yields on this input (blinding r, s: this instance's unless given)."""
        w = limbs_to_ints(self.w)
        dot = lambda ks, ws: sum(a * b for a, b in zip(limbs_to_ints(ks), ws)) % R
        alpha, beta, delta = (limbs_to_ints(k)[0] for k in (self.k_alpha, self.k_beta, self.k_delta))
        r, s = (self.r if r is None else r), (self.s if s is None else s)
        a = (dot(self.k_at, w) + alpha + r * delta) % R
        b = (dot(self.k_b, w) + beta + s * delta) % R
        l1 = self.npublic + 1
        c_msm = dot(self.k_c[l1:], w[l1:])
        h_msm = dot(self.k_ptd[: self.n - 1], limbs_to_ints(self.h0))
        c = (c_msm + h_msm + s * a + r * b - r * s * delta) % R
        return a, b, c

    def algorithmic_bytes(self):
        """SURVEY §8(d): 96 B per G1 term, 160 B per G2 term, each MSM counted independently."""
        m, n = self.m, self.n
        return 96 * m + 96 * m + 160 * m + 96 * (m - 2) + 96 * (n - 1)


class SyntheticCircuit:
    """The synthetic R1CS of SURVEY §8d (configs 2 / 4): n constraints over m = n + 2 signals [one, pub, x_0 .. x_{n-1}],
    a multiplication chain with full-width values:

        (x_0 + 5) * x_0 = x_1;     x_k * x_{k-1} = x_{k+1}  (k = 1 .. n-2);     x_{n-1} * x_{n-2} = pub

    1-2 non-zeros per row of A, one in B, one in C (coefficients 1 and the 5 of README.md:174).  CSR arrays are numpy;
    the witness is the chain evaluated mod r from a seeded x_0 (NPublic = 1: the last product).

    ``short_z=True``: the m = n + 1 variant, n constraints over [one, pub, c_0 .. c_{n-2}] — the linear row c_0 * one = c_0,
    then the n - 1 products of the same chain (c_0 + 5) * c_0 = c_1, c_k * c_{k-1} = c_{k+1}, the last one into pub.  Its
    Z has length m - 1 = n."""

    def __init__(self, n, seed=SEED_WITNESS, short_z=False):
        assert n >= 2
        if short_z:
            self._init_short(n, seed)
            return
        self.n, self.m, self.npublic = n, n + 2, 1
        j = np.arange(n, dtype=np.uint32)
        # A: row 0 = {x_0: 1, one: 5}, row j = {x_j: 1}
        a_rowptr = np.concatenate(([0, 2], 2 + np.arange(1, n, dtype=np.uint32))).astype(np.uint32)
        a_col = np.concatenate(([0, 2], 2 + j[1:])).astype(np.uint32)          # columns sorted inside row 0: one, x_0
        a_val = np.zeros((n + 1, 4), dtype=np.uint64)
        a_val[:, 0] = 1
        a_val[0, 0] = 5
        b_rowptr = np.arange(n + 1, dtype=np.uint32)
        b_col = np.concatenate(([2], 2 + j[1:] - 1)).astype(np.uint32)          # row 0: x_0; row j: x_{j-1}
        c_col = np.concatenate((3 + j[:-1], [1])).astype(np.uint32)             # row j: x_{j+1}; last row: pub
        ones = np.zeros((n, 4), dtype=np.uint64)
        ones[:, 0] = 1
        self.csr = [(a_rowptr, a_col, a_val), (b_rowptr, b_col, ones), (b_rowptr.copy(), c_col, ones.copy())]
        x0 = limbs_to_ints(rand_limbs(1, seed))[0] % R
        xs = [x0, (x0 + 5) * x0 % R]
        for k in range(1, n - 1):
            xs.append(xs[k] * xs[k - 1] % R)
        pub = xs[n - 1] * xs[n - 2] % R
        self.witness = [1, pub] + xs[:n]
        self.public_signals = [pub]

    def _init_short(self, n, seed):
        self.n, self.m, self.npublic = n, n + 1, 1
        j = np.arange(2, n, dtype=np.uint32)                                   # product rows 2 .. n-1
        rowptr1 = np.arange(n + 1, dtype=np.uint32)
        # A: row 0 = {c_0}, row 1 = {one: 5, c_0}, row j = {c_{j-1}};  B: row 0 = {one}, row 1 = {c_0}, row j = {c_{j-2}}
        a_rowptr = np.concatenate(([0, 1], 3 + np.arange(n - 1, dtype=np.uint32))).astype(np.uint32)
        a_col = np.concatenate(([2, 0, 2], j + 1)).astype(np.uint32)
        a_val = np.zeros((n + 1, 4), dtype=np.uint64)
        a_val[:, 0] = 1
        a_val[1, 0] = 5
        b_col = np.concatenate(([0, 2], j)).astype(np.uint32)
        # C: row 0 = {c_0}, row j = {c_j} (j < n-1), row n-1 = {pub}
        c_col = np.concatenate(([2], 2 + np.arange(1, n - 1, dtype=np.uint32), [1])).astype(np.uint32)
        ones = np.zeros((n, 4), dtype=np.uint64)
        ones[:, 0] = 1
        self.csr = [(a_rowptr, a_col, a_val), (rowptr1, b_col, ones), (rowptr1.copy(), c_col, ones.copy())]
        c0 = limbs_to_ints(rand_limbs(1, seed))[0] % R
        cs = [c0, (c0 + 5) * c0 % R]
        for k in range(1, n - 1):
            cs.append(cs[k] * cs[k - 1] % R)
        self.witness = [1, cs[n - 1]] + cs[:n - 1]
        self.public_signals = [cs[n - 1]]

    def dense(self):
        """The same R1CS as dense n x m matrices (small n only): the reference's a, b, c."""
        out = []
        for rowptr, col, val in self.csr:
            vals = limbs_to_ints(val)
            M = [[0] * self.m for _ in range(self.n)]
            for r_ in range(self.n):
                for k in range(int(rowptr[r_]), int(rowptr[r_ + 1])):
                    M[r_][int(col[k])] = vals[k]
            out.append(M)
        return out


class CircuitQAP:
    """What a real trusted setup of SyntheticCircuit(n) starts from, shared by CircuitGroth16 and CircuitPinocchio: the R1CS
    resident on the device, the satisfying witness (limbs in ``w``), Z = prod_{i=1..n}(x - i) (groth16.go:122-132,
    snark.go:210-221), and the QAP evaluated at the toxic T for every signal — at_s / bt_s / ct_s = Eval(alphas[i], T) etc.
    through the sparse A^T l(T) of b200_qap_eval_at, and zt = Z(T) — as Python ints.  Any n >= 2.  ``short_z``: the
    m = n + 1 variant of SyntheticCircuit, whose Z = prod_{i=1..n-1}(x - i) has length m - 1 = n."""

    def __init__(self, n, t, short_z=False):
        from .r1csqap import SparseR1CS
        assert n >= 2
        self.circuit = SyntheticCircuit(n, short_z=short_z)
        self.n, self.m, self.npublic = n, self.circuit.m, 1
        self.short_z = short_z
        self.logn = n.bit_length() - 1 if n & (n - 1) == 0 else None
        self.r1cs = SparseR1CS(n, self.m, self.circuit.csr)
        at_l, bt_l, ct_l, self.zt = self.r1cs.EvalAt(t)                      # zt = Z(T), Z of m - 2 roots
        self.at_s, self.bt_s, self.ct_s = limbs_to_ints(at_l), limbs_to_ints(bt_l), limbs_to_ints(ct_l)
        self.w = ints_to_limbs(self.circuit.witness)
        nz = self.m - 2
        self.z = np.zeros((nz + 1, 4), dtype=np.uint64)
        check(lib().b200_zero_poly(nz, ptr(self.z)))

    def px_of(self, w_limbs):
        """px = A(x) B(x) - C(x) of a witness of this R1CS (r1csqap.go:191-210), from the sparse front end (b200_qap_px)."""
        return self.r1cs.combine_limbs(w_limbs, want_abc=False)[3]


def _size(logn, n):
    assert (logn is None) != (n is None), "give logn or n"
    return 1 << logn if n is None else n


class CircuitGroth16(CircuitQAP, SyntheticGroth16):
    """A REAL Groth16 instance at benchmark sizes: SyntheticCircuit's R1CS, a satisfying witness, and the CRS that
    groth16.GenerateTrustedSetup (groth16/groth16.go:94-222) yields for seeded toxic values — every point is still
    k*G with a known k (k = Eval(alphas[i], tau) etc., see CircuitQAP), so
    the known-discrete-log parity check of SyntheticGroth16 keeps working AND the proof verifies under the real Vk.
    px comes from the sparse QAP front end (b200_qap_px); the expected proof is computed in the exponent from the QAP
    identity  h(tau) Z(tau) = A(tau) B(tau) - C(tau)  — independently of the GPU's px and h.  Sized by 2^logn or by n;
    ``short_z``: the m = n + 1 circuit (len(Z) = n)."""

    def __init__(self, logn=None, mint=True, n=None, short_z=False):
        tox = [x % R for x in limbs_to_ints(rand_limbs(5, SEED_TOXIC))]
        self.toxic = dict(zip(("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta"), tox))
        t, ka, kb, kg, kd = tox
        super().__init__(_size(logn, n), t, short_z)
        m = self.m
        self.n_ptd = m - 1
        at, bt, ct, zt = self.at_s, self.bt_s, self.ct_s, self.zt
        inv_d, inv_g = pow(kd, -1, R), pow(kg, -1, R)
        l1 = self.npublic + 1
        kc = [0] * l1 + [inv_d * ((at[i] * kb + bt[i] * ka + ct[i]) % R) % R for i in range(l1, m)]      # :181-200
        self.k_ic = [inv_g * ((at[i] * kb + bt[i] * ka + ct[i]) % R) % R for i in range(l1)]               # :202-219
        ptd, cur = [], zt * inv_d % R                                                                      # :139-149
        for _ in range(self.n_ptd):
            ptd.append(cur)
            cur = cur * t % R
        self.k_at, self.k_b, self.k_c, self.k_ptd = (ints_to_limbs(v) for v in (at, bt, kc, ptd))
        self.k_alpha, self.k_beta, self.k_delta, self.k_gamma = (ints_to_limbs([v]) for v in (ka, kb, kd, kg))
        rs = limbs_to_ints(rand_limbs(2, SEED_RS))
        self.r, self.s = rs[0] >> 13, rs[1] >> 13
        if mint:
            self.mint()

    def mint(self):
        self.at = mint_points(1, self.k_at)
        self.b1 = mint_points(1, self.k_b)
        self.b2 = mint_points(2, self.k_b)
        self.cd = mint_points(1, self.k_c)
        self.ptd = mint_points(1, self.k_ptd)
        self.alpha1, self.beta1, self.delta1 = (mint_points(1, k) for k in (self.k_alpha, self.k_beta, self.k_delta))
        self.beta2, self.delta2, self.gamma2 = (mint_points(2, k) for k in (self.k_beta, self.k_delta, self.k_gamma))
        self.ic = mint_points(1, ints_to_limbs(self.k_ic))
        self.px = self.px_of(self.w)

    def expected_dlogs(self, witness=None, r=None, s=None):
        """Discrete logs of PiA, PiB, PiC for ``witness`` (ints, a satisfying witness of this R1CS, e.g. of
        SyntheticCircuit(n, seed=...)) and blinding r, s — this instance's own unless given."""
        w = self.circuit.witness if witness is None else witness
        dot = lambda ks: sum(a * b for a, b in zip(ks, w)) % R
        t, ka, kb, kg, kd = (self.toxic[k] for k in ("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta"))
        A, B, C = dot(self.at_s), dot(self.bt_s), dot(self.ct_s)
        r, s = (self.r if r is None else r), (self.s if s is None else s)
        a = (A + ka + r * kd) % R
        b = (B + kb + s * kd) % R
        l1 = self.npublic + 1
        kc = limbs_to_ints(self.k_c)
        c_msm = sum(x * y for x, y in zip(kc[l1:], w[l1:])) % R
        h_msm = (A * B - C) * pow(kd, -1, R) % R                     # sum_i h_i tau^i Z(tau)/delta = (A B - C)(tau)/delta
        c = (c_msm + h_msm + s * a + r * b - r * s * kd) % R
        return a, b, c

    def vk_limbs(self):
        """(ic, alpha1, beta2, gamma2, delta2) as limb arrays for b200_groth16_verify."""
        return self.ic, self.alpha1, self.beta2, self.gamma2, self.delta2

    def verify(self, pi_a, pi_b, pi_c):
        """groth16.VerifyProof (groth16.go:281-305) on the GPU against this instance's real verification key."""
        import ctypes
        ok = ctypes.c_int(0)
        pub = ints_to_limbs(self.circuit.public_signals)
        check(lib().b200_groth16_verify(ptr(self.ic), self.npublic + 1, ptr(self.alpha1), ptr(self.beta2), ptr(self.gamma2),
                                        ptr(self.delta2), ptr(pi_a), ptr(pi_b), ptr(pi_c), ptr(pub), 1, ctypes.byref(ok)))
        return bool(ok.value)


PINOCCHIO_TOXIC = ("T", "Ka", "Kb", "Kc", "Kbeta", "Kgamma", "RhoA", "RhoB")


def pinocchio_toxic(seed=SEED_TOXIC):
    """Seeded toxic values of snark.GenerateTrustedSetup (snark.go:98-251), keyed as its Toxic struct (RhoC is derived)."""
    return dict(zip(PINOCCHIO_TOXIC, (x % R for x in limbs_to_ints(rand_limbs(len(PINOCCHIO_TOXIC), seed)))))


def pinocchio_key_dlogs(at, bt, ct, zt, toxic, npublic):
    """Discrete logs (w.r.t. the generators) of every point of the Pinocchio key and Vk that snark.GenerateTrustedSetup
    (snark.go:98-251) makes from at / bt / ct = Eval(alphas[i], T) etc. over all signals and zt = Z(T).  Pure ints:
    A, Ap, Bp, C, Cp, Kp, G1T and Vkb, G1Kbg are in G1; B and Vka, Vkc, G2Kbg, G2Kg, Vkz in G2; IC = A[0..NPublic]."""
    t, ka, kb, kc, kbeta, kgamma, rho_a, rho_b = (toxic[k] % R for k in PINOCCHIO_TOXIC)
    rho_c = rho_a * rho_b % R                                    # :150
    kbg = kbeta * kgamma % R
    a = [rho_a * x % R for x in at]                              # :171-207
    b = [rho_b * x % R for x in bt]
    c = [rho_c * x % R for x in ct]
    g1t, cur = [], 1                                             # G1T[j] = T^j, j = 0 .. len(Z) - 1 (:230-237)
    for _ in range(len(at) - 1):
        g1t.append(cur)
        cur = cur * t % R
    return {"A": a, "Ap": [ka * x % R for x in a], "B": b, "Bp": [kb * x % R for x in b], "C": c,
            "Cp": [kc * x % R for x in c], "Kp": [kbeta * (x + y + z) % R for x, y, z in zip(a, b, c)], "G1T": g1t,
            "Vka": ka, "Vkb": kb, "Vkc": kc, "G1Kbg": kbg, "G2Kbg": kbg, "G2Kg": kgamma, "Vkz": rho_c * zt % R,
            "IC": a[:npublic + 1]}


def pinocchio_proof_dlogs(at, bt, ct, zt, toxic, npublic, w):
    """Discrete logs of the eight elements snark.GenerateProofs (snark.go:254-289) returns for witness w under the key of
    pinocchio_key_dlogs, from the QAP identity  h(T) Z(T) = A(T) B(T) - C(T)  (A(T) = sum over ALL signals of w_i at_i),
    independently of px and of the quotient h."""
    _, ka, kb, kc, kbeta, _, rho_a, rho_b = (toxic[k] % R for k in PINOCCHIO_TOXIC)
    rho_c = rho_a * rho_b % R
    dot = lambda ks, lo=0: sum(k * x for k, x in zip(ks[lo:], w[lo:])) % R
    A, B, C = dot(at), dot(bt), dot(ct)
    pi_a = rho_a * dot(at, npublic + 1) % R                      # public signals excluded, :265-268
    return {"PiA": pi_a, "PiAp": ka * pi_a % R, "PiB": rho_b * B % R, "PiBp": kb * rho_b * B % R, "PiC": rho_c * C % R,
            "PiCp": kc * rho_c * C % R, "PiH": (A * B - C) * pow(zt, -1, R) % R,
            "PiKp": kbeta * (rho_a * A + rho_b * B + rho_c * C) % R}


class CircuitPinocchio(CircuitQAP):
    """A REAL Pinocchio instance at benchmark sizes (any n >= 2): SyntheticCircuit's R1CS and witness, and the key and Vk
    that snark.GenerateTrustedSetup (snark.go:98-251) yields for seeded toxic values.  Every point is k*G with k from
    pinocchio_key_dlogs, minted on the GPU; the expected proof comes from pinocchio_proof_dlogs.  Key arrays are Jacobian
    limbs in ``pk`` (A, Ap, B (G2), Bp, C, Cp, Kp, G1T), the Vk is a snark.VerifyProof dict of points in ``vk``.
    ``short_z``: the m = n + 1 circuit (len(Z) = len(G1T) = n)."""

    def __init__(self, n, mint=True, short_z=False):
        self.toxic = pinocchio_toxic()
        super().__init__(n, self.toxic["T"], short_z)
        self.k = pinocchio_key_dlogs(self.at_s, self.bt_s, self.ct_s, self.zt, self.toxic, self.npublic)
        if mint:
            self.mint()

    def mint(self):
        from .bn128 import _unflatten_g1, _unflatten_g2
        k = self.k
        self.pk = {s: mint_points(2 if s == "B" else 1, ints_to_limbs(k[s])) for s in ("A", "Ap", "B", "Bp", "C", "Cp", "Kp", "G1T")}
        g1 = ("Vkb", "G1Kbg")
        g2 = ("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz")
        self.vk = dict(zip(g1, _unflatten_g1(mint_points(1, ints_to_limbs([k[s] for s in g1])))))
        self.vk.update(zip(g2, _unflatten_g2(mint_points(2, ints_to_limbs([k[s] for s in g2])))))
        self.vk["IC"] = _unflatten_g1(self.pk["A"][: self.npublic + 1])
        self.px = self.px_of(self.w)

    def load_pk(self, rank=0, world=1, window_bits=0):
        p = self.pk
        h = _lib._h(0)
        check(lib().b200_pinocchio_pk_load_shard(
            ptr(p["A"]), ptr(p["Ap"]), ptr(p["B"]), ptr(p["Bp"]), ptr(p["C"]), ptr(p["Cp"]), ptr(p["Kp"]), self.m,
            ptr(p["G1T"]), p["G1T"].shape[0], ptr(self.z), self.z.shape[0], self.npublic, window_bits, rank, world, h))
        return h.value

    def expected_dlogs(self, witness=None):
        """Discrete logs of PiA .. PiKp, PiB for ``witness`` (ints; this instance's own unless given)."""
        w = self.circuit.witness if witness is None else witness
        return pinocchio_proof_dlogs(self.at_s, self.bt_s, self.ct_s, self.zt, self.toxic, self.npublic, w)

    def verify(self, proof, public=None):
        """snark.VerifyProof (snark.go:292-372) on the GPU against this instance's Vk."""
        from . import snark
        return snark.VerifyProof(self.vk, proof, self.circuit.public_signals if public is None else public)
