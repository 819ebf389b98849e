"""Proofs of witnesses that do NOT satisfy the R1CS, and sparse R1CS of irregular shape.

groth16.GenerateProofs and snark.GenerateProofs prove any witness: they take h = DivisorPolynomial(px, Z) — the quotient,
remainder dropped (groth16.go:266, snark.go:280, r1csqap.go:213-216).  With a_j = (A w)_j and b_j = (B w)_j, the values on
the points 1..n, and deg Z = n:

    h(tau) Z(tau) = A(tau) B(tau) - sum_j a_j b_j l_j(tau)        (l_j: the Lagrange basis of {1..n})

because deg C < n, so quotient(A B - C, Z) = quotient(A B - c', Z) for c' the interpolant of the products a_j b_j, and
A B - c' vanishes on 1..n.  For a satisfying witness c' = C and this is the usual QAP identity.  Every expectation here
comes from it in Python ints — independently of the device's px, h and interpolation — and is held against the oracle's
reference-order prover on the CPU (no GPU needed), then against every Groth16 entry point (px-fed and witness-fed, host
and device, sharded, reduced tables, two contexts in flight) and Pinocchio on the GPU.

The second half feeds the sparse front end (b200_qap_px, b200_qap_eval_at, the witness-fed quotient, the setup's CSC
transpose) R1CS with empty rows, a dense row, explicit zero and r - 1 coefficients, unused columns and a repeated
(row, column) entry, which acts as the sum of its coefficients as in a dense matrix."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

from oracle import ref_py as o

G1, G2 = o.BN.G1, o.BN.G2
R = o.R


# ---- expectations for any witness (Python ints) --------------------------------------------------------------------
def lagrange_at(n, t):
    """[l_j(t)] for j < n, the Lagrange basis of {1..n} at t (t not in 1..n): l_j(t) = Z(t) / ((t - j - 1) d_j) with
    d_j = prod_{i != j} (j - i) = (-1)^(n-1-j) j! (n-1-j)!; one batch inversion."""
    fact = [1] * n
    for i in range(1, n):
        fact[i] = fact[i - 1] * i % R
    den = [(t - j - 1) * fact[j] % R * fact[n - 1 - j] % R for j in range(n)]
    pre = [1] * (n + 1)
    zt = 1
    for j in range(n):
        pre[j + 1] = pre[j] * den[j] % R
        zt = zt * (t - j - 1) % R
    inv = pow(pre[n], -1, R)
    out = [0] * n
    for j in range(n - 1, -1, -1):
        v = zt * inv % R * pre[j] % R
        out[j] = (R - v) % R if (n - 1 - j) & 1 else v
        inv = inv * den[j] % R
    return out


def _ints(val):
    if hasattr(val, "dtype"):
        from gosnark_b200._lib import limbs_to_ints
        return limbs_to_ints(val)
    return [int(x) % R for x in val]


def row_values(csr, w):
    """(M w)_j for every row j of a CSR matrix (rowptr, col, val): a repeated (row, column) entry adds."""
    rowptr, col, val = csr
    rowptr, col, val = [int(x) for x in rowptr], [int(x) for x in col], _ints(val)
    return [sum(val[k] * w[col[k]] for k in range(rowptr[j], rowptr[j + 1])) % R for j in range(len(rowptr) - 1)]


def hz_at(csr3, w, lag, at, bt):
    """h(tau) Z(tau) = A(tau) B(tau) - sum_j a_j b_j l_j(tau) for witness w; at, bt: Eval(alphas[i], tau) etc. per signal."""
    a, b = row_values(csr3[0], w), row_values(csr3[1], w)
    A = sum(x * y for x, y in zip(at, w)) % R
    B = sum(x * y for x, y in zip(bt, w)) % R
    return (A * B - sum(x * y % R * l for x, y, l in zip(a, b, lag))) % R


def satisfied(csr3, w):
    a, b, c = (row_values(M, w) for M in csr3)
    return all(x * y % R == z for x, y, z in zip(a, b, c))


def groth16_dlogs(inst, w, r, s, hz=None):
    """Discrete logs of PiA, PiB, PiC that groth16.GenerateProofs (groth16.go:225-278) returns for ANY witness w under the
    CRS of inst (CircuitGroth16 or a key of the same shape: at_s, bt_s, k_c, toxic, npublic, circuit.csr, lag).
    hz: h(T) Z(T) when len(Z) != n + 1 (hz_at assumes deg Z = n)."""
    from gosnark_b200._lib import limbs_to_ints
    ka, kb, kd = (inst.toxic[k] for k in ("Kalpha", "Kbeta", "Kdelta"))
    A = sum(x * y for x, y in zip(inst.at_s, w)) % R
    B = sum(x * y for x, y in zip(inst.bt_s, w)) % R
    a, b = (A + ka + r * kd) % R, (B + kb + s * kd) % R
    l1 = inst.npublic + 1
    c_msm = sum(x * y for x, y in zip(limbs_to_ints(inst.k_c)[l1:], w[l1:])) % R
    if hz is None:
        hz = hz_at(inst.circuit.csr, w, inst.lag, inst.at_s, inst.bt_s)
    h_msm = hz * pow(kd, -1, R) % R
    return a, b, (c_msm + h_msm + s * a + r * b - r * s * kd) % R


def pinocchio_dlogs(inst, w):
    """snark.GenerateProofs' eight elements for ANY witness w (CircuitPinocchio): pinocchio_proof_dlogs with PiH from the
    quotient with the remainder dropped."""
    from gosnark_b200.synthetic import pinocchio_proof_dlogs
    d = pinocchio_proof_dlogs(inst.at_s, inst.bt_s, inst.ct_s, inst.zt, inst.toxic, inst.npublic, w)
    d["PiH"] = hz_at(inst.circuit.csr, w, inst.lag, inst.at_s, inst.bt_s) * pow(inst.zt, -1, R) % R
    return d


def perturbed(w, how, n, seed=0):
    """Witnesses of SyntheticCircuit-shaped signals [one, pub, x_0 .. x_{n-1}] that break some rows of the chain."""
    w = list(w)
    if how == "public":                 # only the last row (x_{n-1} x_{n-2} = pub) is off
        w[1] = (w[1] + 1) % R
    elif how == "x0":                   # rows 0 and 1
        w[2] = (w[2] + 1) % R
    elif how == "middle":               # the rows around n/2 (a power-of-two boundary of the interpolation at 2^k + 2)
        w[2 + n // 2] = (w[2 + n // 2] + 7) % R
    elif how == "random":               # almost every row
        rng = random.Random(seed)
        w = [1] + [rng.randrange(R) for _ in range(len(w) - 1)]
    elif how == "one2":                 # the signal "one" is 2: row 0's constant term doubles
        w[0] = 2
    else:
        raise ValueError(how)
    return w


HOWS = ("public", "x0", "middle", "random", "one2")


# ---- CPU: the expectation against the oracle's reference-order provers ----------------------------------------------
def _dense_toxic_instance(n):
    """SyntheticCircuit(n) as the reference's dense matrices, its QAP (R1CSToQAP) and seeded toxic values."""
    from gosnark_b200.synthetic import SyntheticCircuit
    circ = SyntheticCircuit(n)
    a, b, c = circ.dense()
    alphas, betas, gammas, z = o.PF.r1cs_to_qap(a, b, c)
    rng = random.Random(0x70C + n)
    return circ, (a, b, c), (alphas, betas, gammas, z), rng


@pytest.mark.parametrize("n", [2, 3, 5])
def test_expectation_matches_reference_groth16_on_unsatisfied_witnesses(n):
    """groth16_dlogs for witnesses that break one, several or all rows == the oracle's GenerateProofs on the same CRS, with
    px from its CombinePolynomials; for the satisfying witness the identity reduces to h(tau) Z(tau) = A B - C."""
    circ, abc, (alphas, betas, gammas, z), rng = _dense_toxic_instance(n)
    m = circ.m
    tox = dict(zip(("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta"), (rng.randrange(n + 1, R) for _ in range(5))))
    pk, _ = o.groth16_setup(m, circ.npublic, alphas, betas, gammas, tox)
    t, kb, ka, kd = tox["T"], tox["Kbeta"], tox["Kalpha"], tox["Kdelta"]

    class Inst:
        pass
    inst = Inst()
    inst.toxic, inst.npublic, inst.circuit = tox, circ.npublic, circ
    inst.at_s = [o.PF.eval(p, t) for p in alphas]
    inst.bt_s = [o.PF.eval(p, t) for p in betas]
    ct = [o.PF.eval(p, t) for p in gammas]
    from gosnark_b200._lib import ints_to_limbs
    inst.k_c = ints_to_limbs([0] * 2 + [pow(kd, -1, R) * (inst.at_s[i] * kb + inst.bt_s[i] * ka + ct[i]) % R
                                        for i in range(2, m)])
    inst.lag = lagrange_at(n, t)
    zt = o.PF.eval(z, t)
    w0 = circ.witness
    assert satisfied(circ.csr, w0)
    C = sum(x * y for x, y in zip(ct, w0)) % R
    A = sum(x * y for x, y in zip(inst.at_s, w0)) % R
    B = sum(x * y for x, y in zip(inst.bt_s, w0)) % R
    assert hz_at(circ.csr, w0, inst.lag, inst.at_s, inst.bt_s) == (A * B - C) % R
    r, s = rng.randrange(R), rng.randrange(R)
    for how in ("satisfied",) + HOWS:
        w = w0 if how == "satisfied" else perturbed(w0, how, n, seed=n)
        assert satisfied(circ.csr, w) == (how == "satisfied"), how
        px = o.PF.combine_polynomials(w, alphas, betas, gammas)[3]
        ref, raw = o.groth16_prove(m, circ.npublic, pk, w, px, r, s)
        hx = raw["hx"]
        assert o.PF.eval(hx, t) * zt % R == hz_at(circ.csr, w, inst.lag, inst.at_s, inst.bt_s), how
        for key, G, d in zip(("PiA", "PiB", "PiC"), (G1, G2, G1), groth16_dlogs(inst, w, r, s)):
            assert G.affine(ref[key]) == G.affine(G.mul_scalar(G.G, d)), (how, key)


@pytest.mark.parametrize("n", [2, 4])
def test_expectation_matches_reference_pinocchio_on_unsatisfied_witnesses(n):
    """pinocchio_dlogs' PiH for unsatisfied witnesses == the oracle's snark.GenerateProofs on the same key."""
    from gosnark_b200.synthetic import pinocchio_toxic
    circ, abc, (alphas, betas, gammas, z), _ = _dense_toxic_instance(n)
    m = circ.m
    tox = pinocchio_toxic()
    pk, _ = o.pinocchio_setup(m, circ.npublic, alphas, betas, gammas, tox)
    pk["Z"] = z

    class Inst:
        pass
    inst = Inst()
    t = tox["T"]
    inst.toxic, inst.npublic, inst.circuit = tox, circ.npublic, circ
    inst.at_s, inst.bt_s, inst.ct_s = ([o.PF.eval(p, t) for p in ps] for ps in (alphas, betas, gammas))
    inst.zt, inst.lag = o.PF.eval(z, t), lagrange_at(n, t)
    for how in ("satisfied", "public", "x0", "random", "one2"):
        w = circ.witness if how == "satisfied" else perturbed(circ.witness, how, n, seed=3)
        px = o.PF.combine_polynomials(w, alphas, betas, gammas)[3]
        ref, _ = o.pinocchio_prove(m, circ.npublic, pk, w, px)
        assert G1.affine(ref["PiH"]) == G1.affine(G1.mul_scalar(G1.G, pinocchio_dlogs(inst, w)["PiH"])), how


def test_lagrange_basis_against_the_interpolation():
    """lagrange_at against the oracle's LagrangeInterpolation evaluated at t (n up to 9, t far from and next to 1..n)."""
    rng = random.Random(11)
    for n in (1, 2, 5, 9):
        v = [rng.randrange(R) for _ in range(n)]
        poly = o.PF.lagrange_interpolation(v)
        for t in (0, n + 1, R - 1, rng.randrange(R)):
            assert sum(x * y for x, y in zip(v, lagrange_at(n, t))) % R == o.PF.eval(poly, t), (n, t)


# ---- GPU helpers ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


def limbs(v):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs([v])


def to_dev(arr):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def split(words):
    """48 u64 (PiA | PiC | PiB) -> affine (PiA, PiB, PiC)."""
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    pa, pc = _unflatten_g1(words[:24])
    return G1.affine(pa), G2.affine(_unflatten_g2(words[24:48])[0]), G1.affine(pc)


def host_words(fn, *args):
    from gosnark_b200._lib import check, ptr
    pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
    check(fn(*args, ptr(pa), ptr(pb), ptr(pc)))
    return np.concatenate([pa, pc, pb])


def expected_points(dlogs):
    a, b, c = dlogs
    return G1.affine(G1.mul_scalar(G1.G, a)), G2.affine(G2.mul_scalar(G2.G, b)), G1.affine(G1.mul_scalar(G1.G, c))


def assert_proof(got, exp, what):
    for name, g, e in zip(("PiA", "PiB", "PiC"), got, exp):
        assert g == e, f"{what}: {name}"


def verifies(L, inst, words, public):
    """b200_groth16_verify of a 48-word proof under inst's real Vk with the given public signals."""
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    words = np.asarray(words, dtype=np.uint64)
    ok = ctypes.c_int(0)
    pa, pc, pb = (np.ascontiguousarray(x) for x in (words[:12], words[12:24], words[24:48]))
    check(L.b200_groth16_verify(ptr(inst.ic), inst.npublic + 1, ptr(inst.alpha1), ptr(inst.beta2), ptr(inst.gamma2),
                                ptr(inst.delta2), ptr(pa), ptr(pb), ptr(pc), ptr(ints_to_limbs(public)), len(public),
                                ctypes.byref(ok)))
    return bool(ok.value)


def load_pk(L, inst, ctx=0, acc=0, rank=0, world=1, t=0):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    try:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, ctx))
        check(L.b200_config(_lib.CFG_ACC_MODE, acc))
        with _lib.table_windows(t):
            return inst.load_pk(rank, world)
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))
        check(L.b200_config(_lib.CFG_ACC_MODE, 0))


def all_entries(L, inst, pk, w_ints, r, s):
    """The same proof through b200_groth16_prove (px from b200_qap_px), b200_groth16_prove_device, b200_groth16_prove_witness
    and b200_groth16_prove_witness_device on a torch side stream: name -> 48 words."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    w = ints_to_limbs(w_ints)
    px = inst.px_of(w)
    h, m, rr, ss = inst.r1cs.handle, inst.m, limbs(r), limbs(s)
    out = {"px-host": host_words(L.b200_groth16_prove, pk, ptr(w), m, ptr(px), px.shape[0], ptr(rr), ptr(ss)),
           "witness-host": host_words(L.b200_groth16_prove_witness, pk, h, ptr(w), m, ptr(rr), ptr(ss))}
    d_out = torch.full((96,), -1, dtype=torch.int64, device="cuda")
    d_w, d_px = to_dev(w), to_dev(px)          # synchronises: the library's stream is not ordered with torch's
    check(L.b200_groth16_prove_device(pk, d_w.data_ptr(), m, d_px.data_ptr(), px.shape[0], ptr(rr), ptr(ss),
                                      d_out.data_ptr(), None))
    torch.cuda.synchronize()                   # two proofs on one prove context must be ordered by the caller
    side = torch.cuda.Stream()
    check(L.b200_groth16_prove_witness_device(pk, h, d_w.data_ptr(), m, ptr(rr), ptr(ss), d_out[48:].data_ptr(),
                                              side.cuda_stream))
    torch.cuda.synchronize()
    words = d_out.cpu().numpy().view(np.uint64)
    out["px-device"], out["witness-device"] = words[:48].copy(), words[48:].copy()
    return out


_instances = {}


def groth16_instance(n):
    """CircuitGroth16 of n constraints (m = n + 2, len(Z) = n + 1: the h-direct branch) with its Lagrange basis at T."""
    from gosnark_b200.synthetic import CircuitGroth16
    key = ("groth16", n)
    if key not in _instances:
        inst = CircuitGroth16(n=n)
        inst.lag = lagrange_at(n, inst.toxic["T"])
        _instances[key] = inst
    return _instances[key]


def pinocchio_instance(n):
    from gosnark_b200.synthetic import CircuitPinocchio
    key = ("pinocchio", n)
    if key not in _instances:
        inst = CircuitPinocchio(n)
        inst.lag = lagrange_at(n, inst.toxic["T"])
        _instances[key] = inst
    return _instances[key]


# ---- GPU a: exact against the oracle at small sizes ------------------------------------------------------------------
def _seeded_dense_key(a, b, c, m, npublic, seed):
    """groth16.GenerateTrustedSetup on dense matrices for seeded toxic values, the points minted on the device by the
    reference-order MulScalar (X,Y,Z-exact): (pk dict, alphas, betas, gammas)."""
    from gosnark_b200._lib import ints_to_limbs
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    from gosnark_b200.synthetic import mint_points
    alphas, betas, gammas, z = o.PF.r1cs_to_qap(a, b, c)
    rng = random.Random(seed)
    t, ka, kb, kg, kd = (rng.randrange(len(a) + 1, R) for _ in range(5))
    ev = lambda ps: [o.PF.eval(p, t) for p in ps]
    at, bt, ct = ev(alphas), ev(betas), ev(gammas)
    zt = o.PF.eval(z, t)
    kc = [0] * (npublic + 1) + [pow(kd, -1, R) * (at[i] * kb + bt[i] * ka + ct[i]) % R for i in range(npublic + 1, m)]
    ptd = [zt * pow(kd, -1, R) * pow(t, i, R) % R for i in range(len(z))]
    g1 = lambda ks: _unflatten_g1(mint_points(1, ints_to_limbs(ks)))
    g2 = lambda ks: _unflatten_g2(mint_points(2, ints_to_limbs(ks)))
    one1, one2 = g1([ka, kb, kd]), g2([kb, kd])
    pk = {"Z": z, "BACDelta": [(0, 0, 0) if k == 0 else p for k, p in zip(kc, g1(kc))], "PowersTauDelta": g1(ptd),
          "G1": {"Alpha": one1[0], "Beta": one1[1], "Delta": one1[2], "At": g1(at), "BACGamma": g1(bt)},
          "G2": {"Beta": one2[0], "Delta": one2[1], "BACGamma": g2(bt)}}
    return pk, alphas, betas, gammas


def _small_cases(golden_dir):
    """(name, dense a | b | c, m, npublic, satisfying witness) for SyntheticCircuit(2 | 5 | 21) and three golden circuits."""
    from gosnark_b200.bn128 import reduce_scalar
    from gosnark_b200.synthetic import SyntheticCircuit
    for n in (2, 5, 21):
        circ = SyntheticCircuit(n)
        yield f"synthetic{n}", circ.dense(), circ.m, circ.npublic, circ.witness
    for name in ("x3x5", "chain21", "mul"):
        with open(os.path.join(golden_dir, f"gobin_{name}.json")) as f:
            g = json.load(f)
        cc = g["compiledcircuit"]
        abc = [[[int(x) % R for x in row] for row in cc["R1CS"][k]] for k in ("A", "B", "C")]
        yield name, abc, cc["NVars"], cc["NPublic"], [reduce_scalar(x) % R for x in g["witness"]]


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_small_circuits_exact_against_the_oracle(L, golden_dir):
    """SyntheticCircuit(2 | 5 | 21) (m = n + 2, the h-direct branch) and the Go binary's x3x5 and chain21 (m = n + 1,
    len(Z) = n: px then the division) and mul (len(Z) = n + 1, h-direct), each on a seeded-toxic key: for witnesses that
    break the last row, the first rows, or every row, b200_groth16_prove with px from CombinePolynomials, the host witness
    entry and the device witness entry all return the affine points of the oracle's GenerateProofs."""
    import torch
    from gosnark_b200 import groth16
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    from gosnark_b200.r1csqap import SparseR1CS
    aff = lambda p: (G1.affine(p["PiA"]), G2.affine(p["PiB"]), G1.affine(p["PiC"]))
    for name, (a, b, c), m, npublic, w0 in _small_cases(golden_dir):
        n = len(a)
        pk, alphas, betas, gammas = _seeded_dense_key(a, b, c, m, npublic, seed=0x5EED0002 + n)
        assert (len(pk["Z"]) == n + 1) == (name not in ("x3x5", "chain21")), name
        sp = SparseR1CS(n, m, (a, b, c))
        csr = [SparseR1CS.dense_to_csr(M) for M in (a, b, c)]
        assert satisfied(csr, w0), name
        dpk = groth16.DeviceProvingKey(pk, m, npublic)
        try:
            rng = random.Random(n)
            bad_last, bad_first = list(w0), list(w0)
            bad_last[npublic] = (bad_last[npublic] + 1) % R
            bad_first[npublic + 1] = (bad_first[npublic + 1] + 3) % R
            wits = {"last": bad_last, "first": bad_first, "random": [1] + [rng.randrange(R) for _ in range(m - 1)]}
            for how, w in wits.items():
                assert not satisfied(csr, w), (name, how)
                r, s = rng.randrange(R), rng.randrange(R)
                px = o.PF.combine_polynomials(w, alphas, betas, gammas)[3]
                exp = aff(o.groth16_prove(m, npublic, pk, w, px, r, s)[0])
                wl = ints_to_limbs(w)
                d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
                check(L.b200_groth16_prove_witness_device(dpk.handle, sp.handle, to_dev(wl).data_ptr(), m, ptr(limbs(r)),
                                                          ptr(limbs(s)), d_out.data_ptr(), None))
                torch.cuda.synchronize()
                got = {"px": aff(dpk.prove_limbs(wl, ints_to_limbs(px), r, s)),
                       "witness-host": aff(dpk.prove_witness_limbs(sp, wl, r, s)),
                       "witness-device": split(d_out.cpu().numpy().view(np.uint64))}
                for entry, p in got.items():
                    assert_proof(p, exp, f"{name} {how} {entry}")
        finally:
            dpk.free()
            sp.free()


# ---- GPU b: benchmark shapes ------------------------------------------------------------------------------------------
def _check_witnesses(L, inst, pk, hows, rs_seed):
    """Every entry point on every witness of `hows`: the §-identity proof, and the GPU verify rejects it."""
    rng = random.Random(rs_seed)
    for how in hows:
        w = perturbed(inst.circuit.witness, how, inst.n, seed=rs_seed)
        r, s = rng.randrange(1 << 240), rng.randrange(1 << 240)
        exp = expected_points(groth16_dlogs(inst, w, r, s))
        got = all_entries(L, inst, pk, w, r, s)
        for entry, words in got.items():
            assert_proof(split(words), exp, f"n={inst.n} {how} {entry}")
        assert not verifies(L, inst, got["witness-device"], [w[1]]), how


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("n,acc", [((1 << 12) + 2, 1), ((1 << 12) + 2, 2), (1 << 16, 1), (1 << 16, 2), (1 << 20, 0)],
                         ids=["4098-affine", "4098-xyzz", "65536-affine", "65536-xyzz", "2^20-auto"])
def test_unsatisfied_witnesses_at_benchmark_sizes(L, n, acc):
    """CircuitGroth16 with the public signal changed, x_0 changed, the rows around n/2 broken, a uniformly random witness
    and one = 2: px-fed (host, device) and witness-fed (host, device on a side stream) proofs all equal the known-dlog
    proof of the quotient with the remainder dropped, and none verifies with its own public signal.  The satisfying
    witness still gives the old expectation and verifies."""
    from gosnark_b200._lib import check
    inst = groth16_instance(n)
    pk = load_pk(L, inst, acc=acc)
    try:
        _check_witnesses(L, inst, pk, HOWS, rs_seed=n + acc)
        w = inst.circuit.witness
        assert groth16_dlogs(inst, w, inst.r, inst.s) == inst.expected_dlogs()
        got = all_entries(L, inst, pk, w, inst.r, inst.s)["witness-device"]
        assert_proof(split(got), expected_points(inst.expected_dlogs()), "satisfied")
        assert verifies(L, inst, got, inst.circuit.public_signals)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [2, 3])
def test_unsatisfied_sharded_emulated(L, world):
    """Every rank's b200_groth16_prove_witness_device record, summed by b200_groth16_finalize_device, is the known-dlog
    proof of an unsatisfied witness (the ranks that hold PowersTauDelta indices run the quotient)."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    inst = groth16_instance((1 << 12) + 2)
    pks = [load_pk(L, inst, rank=rk, world=world) for rk in range(world)]
    try:
        for how in ("middle", "random"):
            w = perturbed(inst.circuit.witness, how, inst.n, seed=world)
            d_w = to_dev(ints_to_limbs(w))
            parts = torch.zeros(128 * world, dtype=torch.int64, device="cuda")
            d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            for rk, pk in enumerate(pks):
                check(L.b200_groth16_prove_witness_device(pk, inst.r1cs.handle, d_w.data_ptr(), inst.m, ptr(limbs(inst.r)),
                                                          ptr(limbs(inst.s)), parts[128 * rk:].data_ptr(), None))
            check(L.b200_groth16_finalize_device(pks[0], parts.data_ptr(), world, ptr(limbs(inst.r)), ptr(limbs(inst.s)),
                                                 d_out.data_ptr(), None))
            torch.cuda.synchronize()
            assert_proof(split(d_out.cpu().numpy().view(np.uint64)), expected_points(groth16_dlogs(inst, w, inst.r, inst.s)),
                         f"world {world} {how}")
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_unsatisfied_on_a_one_window_table_key(L):
    """A key with one stored window row per base set (B200_CFG_TABLE_WINDOWS = 1): every entry point, two witnesses."""
    from gosnark_b200._lib import check
    inst = groth16_instance((1 << 12) + 2)
    pk = load_pk(L, inst, t=1)
    try:
        _check_witnesses(L, inst, pk, ("x0", "random"), rs_seed=1)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_two_contexts_in_flight_satisfied_and_not(L):
    """Keys of contexts 0 and 1 on one R1CS handle, both proofs enqueued before either is waited for: context 0 proves the
    satisfying witness, context 1 one that breaks the middle rows, then the other way round.  Each proof matches its own
    expectation, so neither context's quotient leaks into the other's."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    inst = groth16_instance((1 << 12) + 2)
    pks = [load_pk(L, inst, ctx=k) for k in range(2)]
    wits = [inst.circuit.witness, perturbed(inst.circuit.witness, "middle", inst.n)]
    d_w = [to_dev(ints_to_limbs(w)) for w in wits]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    try:
        for rnd in range(2):
            outs = [torch.zeros(48, dtype=torch.int64, device="cuda") for _ in range(2)]
            torch.cuda.synchronize()
            for k in range(2):
                check(L.b200_groth16_prove_witness_device(pks[k], inst.r1cs.handle, d_w[(k + rnd) % 2].data_ptr(), inst.m,
                                                          ptr(limbs(inst.r)), ptr(limbs(inst.s)), outs[k].data_ptr(),
                                                          streams[k].cuda_stream))
            torch.cuda.synchronize()
            for k in range(2):
                exp = expected_points(groth16_dlogs(inst, wits[(k + rnd) % 2], inst.r, inst.s))
                assert_proof(split(outs[k].cpu().numpy().view(np.uint64)), exp, f"round {rnd} context {k}")
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


# ---- GPU c: Pinocchio ------------------------------------------------------------------------------------------------
P_ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


def _pinocchio_affine(g1, pb):
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    d = {k: G1.affine(p) for k, p in zip(P_ORDER, _unflatten_g1(g1))}
    d["PiB"] = G2.affine(_unflatten_g2(pb)[0])
    return d


def _pinocchio_expected(d):
    e = {k: G1.affine(G1.mul_scalar(G1.G, d[k])) for k in P_ORDER}
    e["PiB"] = G2.affine(G2.mul_scalar(G2.G, d["PiB"]))
    return e


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [(1 << 12) + 2, 1 << 16], ids=["4098", "65536"])
def test_pinocchio_unsatisfied(L, n):
    """b200_pinocchio_prove on px of unsatisfied witnesses, and (at 2^12 + 2) the world-3 records summed by
    b200_pinocchio_finalize_records: all eight elements equal the known-dlog proof with PiH of the quotient."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    inst = pinocchio_instance(n)
    pk = inst.load_pk()
    world = 3
    shards = [inst.load_pk(rk, world) for rk in range(world)] if n < (1 << 16) else []
    try:
        for how in ("public", "middle", "random", "one2"):
            w = perturbed(inst.circuit.witness, how, n, seed=n)
            wl = ints_to_limbs(w)
            px = inst.px_of(wl)
            exp = _pinocchio_expected(pinocchio_dlogs(inst, w))
            g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
            check(L.b200_pinocchio_prove(pk, ptr(wl), inst.m, ptr(px), px.shape[0], ptr(g1), ptr(pb)))
            assert _pinocchio_affine(g1, pb) == exp, how
            if shards:
                recs = torch.zeros(256 * world, dtype=torch.int64, device="cuda")
                torch.cuda.synchronize()
                for rk, spk in enumerate(shards):
                    check(L.b200_pinocchio_prove_record_device(spk, ptr(wl), inst.m, ptr(px), px.shape[0],
                                                               recs[256 * rk:].data_ptr()))
                g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
                check(L.b200_pinocchio_finalize_records(recs.data_ptr(), world, ptr(g1), ptr(pb)))
                assert _pinocchio_affine(g1, pb) == exp, (how, "records")
    finally:
        for k in [pk] + shards:
            check(L.b200_pk_free(k))


# ---- GPU d: irregular sparse R1CS ------------------------------------------------------------------------------------
class IrregularR1CS:
    """A seeded sparse R1CS over m signals [one, pub, x_0 ..] with n constraints that is satisfiable by construction:
      - A and B rows with 0 .. 3 terms, some EMPTY; one A row and one B row of ~512 terms;
      - explicit 0 and r - 1 coefficients; a repeated (row, column) entry in A, B and C (acts as the sum);
      - every C row holds `one`, and one column k with coefficient (a_j b_j - rest_j) / w_k, so row j holds;
      - the last few private columns are used by no matrix.
    Rows are listed with columns in any order (the loader keeps them as given)."""

    def __init__(self, n, m, seed):
        rng = random.Random(seed)
        self.n, self.m, self.npublic = n, m, 1
        unused = set(range(m - 5, m))
        used = [i for i in range(2, m) if i not in unused]
        pool_ab, pool_c = used + [0, 1], used + [1]
        w = [1, rng.randrange(1, R)] + [rng.randrange(1, R) for _ in range(m - 2)]
        self.witness = w
        coef = lambda: rng.choice([0, R - 1, 1, 2, rng.randrange(R), rng.randrange(R)])
        rows = {"A": [], "B": [], "C": []}
        dense_a, dense_b = n // 2, n // 3
        for j in range(n):
            for M, dense in (("A", dense_a), ("B", dense_b)):
                if j == dense:
                    cols = rng.sample(used, min(512, len(used)))
                elif j % 7 == (3 if M == "A" else 5):
                    cols = []                                     # empty row
                else:
                    cols = [rng.choice(pool_ab) for _ in range(rng.randrange(1, 4))]
                rows[M].append([(c, coef()) for c in cols])
        rows["A"][1] += [(rows["A"][1][0][0], 5)] if rows["A"][1] else []
        rows["B"][2] += [(rows["B"][2][0][0], R - 3)] if rows["B"][2] else []
        self.csr = []
        for M in ("A", "B"):
            self.csr.append(self._csr(rows[M]))
        a, b = row_values(self.csr[0], w), row_values(self.csr[1], w)
        for j in range(n):
            row = [(0, coef())] + [(rng.choice(pool_c), coef()) for _ in range(rng.randrange(0, 3))]
            if j == 4:
                row.append(row[0])                                # the repeated (row, column) entry
            k = used[(j * 7919) % len(used)]
            rest = sum(v * w[cc] for cc, v in row) % R
            row.append((k, (a[j] * b[j] - rest) * pow(w[k], -1, R) % R))
            rng.shuffle(row)
            rows["C"].append(row)
        self.csr.append(self._csr(rows["C"]))
        self.rows = rows
        self.public_signals = [w[1]]
        assert satisfied(self.csr, w)

    @staticmethod
    def _csr(rows):
        rowptr = np.zeros(len(rows) + 1, dtype=np.uint32)
        rowptr[1:] = np.cumsum([len(r) for r in rows])
        col = np.array([c for r in rows for c, _ in r], dtype=np.uint32)
        return rowptr, col, [v for r in rows for _, v in r]

    def eval_at(self, t):
        """at / bt / ct of every signal: sum over each matrix's entries (j, i, v) of v l_j(t) — the dense Eval(alphas[i], t)."""
        lag = lagrange_at(self.n, t)
        outs = []
        for rowptr, col, val in self.csr:
            o_ = [0] * self.m
            for j in range(self.n):
                for k in range(int(rowptr[j]), int(rowptr[j + 1])):
                    o_[int(col[k])] = (o_[int(col[k])] + val[k] * lag[j]) % R
            outs.append(o_)
        return outs, lag


class IrregularGroth16:
    """The CRS of groth16.GenerateTrustedSetup for an IrregularR1CS, minted from at / bt / ct computed in PYTHON (so the
    device's b200_qap_eval_at is checked against them, not used)."""

    def __init__(self, n, m, seed):
        from gosnark_b200._lib import check, ints_to_limbs, lib, ptr
        from gosnark_b200.r1csqap import SparseR1CS
        from gosnark_b200.synthetic import mint_points
        self.n, self.m, self.npublic = n, m, 1
        self.circuit = IrregularR1CS(n, m, seed)
        self.r1cs = SparseR1CS(n, m, self.circuit.csr)
        rng = random.Random(seed + 1)
        self.toxic = dict(zip(("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta"), (rng.randrange(n + 1, R) for _ in range(5))))
        t, ka, kb, kg, kd = (self.toxic[k] for k in ("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta"))
        (self.at_s, self.bt_s, self.ct_s), self.lag = self.circuit.eval_at(t)
        nz = m - 2                                   # Z = prod_{i=1..m-2} (x - i) (groth16.go:122-132)
        self.z = np.zeros((nz + 1, 4), dtype=np.uint64)
        check(lib().b200_zero_poly(nz, ptr(self.z)))
        zt = 1
        for i in range(1, nz + 1):
            zt = zt * (t - i) % R
        self.zt = zt
        l1 = self.npublic + 1
        inv_d, inv_g = pow(kd, -1, R), pow(kg, -1, R)
        kc = [0] * l1 + [inv_d * ((self.at_s[i] * kb + self.bt_s[i] * ka + self.ct_s[i]) % R) % R for i in range(l1, m)]
        k_ic = [inv_g * ((self.at_s[i] * kb + self.bt_s[i] * ka + self.ct_s[i]) % R) % R for i in range(l1)]
        ptd = [zt * inv_d % R * pow(t, i, R) % R for i in range(m - 1)]
        self.k_c = ints_to_limbs(kc)
        self.at, self.b1, self.cd, self.ptd = (mint_points(1, ints_to_limbs(v)) for v in (self.at_s, self.bt_s, kc, ptd))
        self.b2 = mint_points(2, ints_to_limbs(self.bt_s))
        self.alpha1, self.beta1, self.delta1 = (mint_points(1, ints_to_limbs([v])) for v in (ka, kb, kd))
        self.beta2, self.delta2, self.gamma2 = (mint_points(2, ints_to_limbs([v])) for v in (kb, kd, kg))
        self.ic = mint_points(1, ints_to_limbs(k_ic))
        self.r, self.s = rng.randrange(1 << 240), rng.randrange(1 << 240)

    def px_of(self, w_limbs):
        return self.r1cs.combine_limbs(w_limbs, want_abc=False)[3]

    def load_pk(self, rank=0, world=1):
        from gosnark_b200 import _lib
        from gosnark_b200._lib import check, lib, ptr
        h = _lib._h(0)
        check(lib().b200_groth16_pk_load_shard(
            ptr(self.at), ptr(self.b1), ptr(self.b2), ptr(self.cd), self.m, ptr(self.ptd), self.m - 1, ptr(self.z),
            self.z.shape[0], ptr(self.alpha1), ptr(self.beta1), ptr(self.delta1), ptr(self.beta2), ptr(self.delta2),
            self.npublic, 0, rank, world, h))
        return h.value

    def dlogs(self, w, r, s):
        """groth16_dlogs for len(Z) = n + 1; for a longer Z (m > n + 2) the remainder is no longer the interpolant of the
        row values, so h(T) Z(T) comes from the device's px (checked against the row values at random points by the test)
        divided by Z in Python."""
        if self.z.shape[0] == self.n + 1:
            return groth16_dlogs(self, w, r, s)
        from gosnark_b200._lib import ints_to_limbs, limbs_to_ints
        rem = limbs_to_ints(self.px_of(ints_to_limbs(w)))
        z = limbs_to_ints(self.z)                   # monic
        h = [0] * (len(rem) - len(z) + 1)
        for k in range(len(h) - 1, -1, -1):         # long division (r1csqap.go:70-84), remainder dropped
            h[k] = q = rem[k + len(z) - 1]
            for i, zi in enumerate(z):
                rem[k + i] = (rem[k + i] - q * zi) % R
        return groth16_dlogs(self, w, r, s, hz=_horner(h, self.toxic["T"]) * self.zt % R)


def _horner(c, x):
    acc = 0
    for v in reversed(c):
        acc = (acc * x + v) % R
    return acc


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("n,m", [((1 << 12) + 2, (1 << 12) + 4), (1 << 16, (1 << 16) + 2), (300, 303)],
                         ids=["4098", "65536", "300-m=n+3"])
def test_irregular_sparse_r1cs(L, n, m):
    """b200_qap_eval_at == the Python A^T l(T) for every signal (repeats summed, unused columns 0); b200_qap_px's ax, bx,
    cx, px at 8 random points == the Python row values' interpolants; and proofs through b200_groth16_prove (px) and both
    witness entries on the CRS minted from the Python at / bt / ct equal the known-dlog proof for the satisfying witness
    (which verifies under the real Vk) and for two unsatisfied ones.  m = n + 3 gives len(Z) = n + 2: the witness entry
    goes through px and the key's division."""
    from gosnark_b200._lib import check, ints_to_limbs, limbs_to_ints
    inst = IrregularGroth16(n, m, seed=n ^ 0xA5A5)
    try:
        circ = inst.circuit
        at_l, bt_l, ct_l, zt = inst.r1cs.EvalAt(inst.toxic["T"])
        assert limbs_to_ints(at_l) == inst.at_s and limbs_to_ints(bt_l) == inst.bt_s and limbs_to_ints(ct_l) == inst.ct_s
        assert zt == inst.zt
        assert all(inst.at_s[i] == inst.bt_s[i] == inst.ct_s[i] == 0 for i in range(m - 5, m))
        w_bad = list(circ.witness)
        w_bad[2] = (w_bad[2] + 1) % R
        rng = random.Random(n)
        w_rand = [1] + [rng.randrange(R) for _ in range(m - 1)]
        assert not satisfied(circ.csr, w_bad) and not satisfied(circ.csr, w_rand)
        for w in (circ.witness, w_bad, w_rand):
            ax, bx, cx, px = (limbs_to_ints(x) for x in inst.r1cs.combine_limbs(ints_to_limbs(w)))
            vals = [row_values(M, w) for M in circ.csr]
            for _ in range(8):
                t = rng.randrange(R)
                lag = lagrange_at(n, t)
                ev = [sum(v * l for v, l in zip(vs, lag)) % R for vs in vals]
                assert [_horner(ax, t), _horner(bx, t), _horner(cx, t)] == ev
                assert _horner(px, t) == (ev[0] * ev[1] - ev[2]) % R
        pk = load_pk(L, inst)
        try:
            for label, w in (("satisfied", circ.witness), ("x0+1", w_bad), ("random", w_rand)):
                exp = expected_points(inst.dlogs(w, inst.r, inst.s))
                got = all_entries(L, inst, pk, w, inst.r, inst.s)
                for entry, words in got.items():
                    assert_proof(split(words), exp, f"{label} {entry}")
                # with len(Z) = n + 2, Z has the root n + 1 where a satisfied a b - c need not vanish: no proof verifies
                assert verifies(L, inst, got["witness-device"], [w[1]]) == (label == "satisfied" and m == n + 2), label
        finally:
            check(L.b200_pk_free(pk))
    finally:
        inst.r1cs.free()
