"""GPU: batched witness-fed Groth16 proving (include/b200snark.h: b200_groth16_prove_witness_batch,
b200_groth16_prove_witness_batch_device): k proofs under one key in one set of launches.

Unless a test says otherwise, every proof p of a batch is checked three ways: it is the known-discrete-log proof of
CircuitGroth16 for (w_p, r_p, s_p) (groth16.GenerateProofs in the exponent), it is the affine proof that
b200_groth16_prove_witness_device gives for the same triple, and a satisfying witness's proof verifies under the real Vk
with that witness's own public signal."""
import ctypes
import json
import os
import threading

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
G1, G2 = o.BN.G1, o.BN.G2
R = o.R
EINVAL, ERANGE = -3, -4


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


_circuits = {}


def circuit(n):
    """CircuitGroth16 of n constraints (len(Z) = n + 1: the h-direct branch), minted once per module."""
    from gosnark_b200.synthetic import CircuitGroth16
    if n not in _circuits:
        _circuits[n] = CircuitGroth16(n=n)
    return _circuits[n]


def witnesses(n, k, seed=0):
    """k distinct satisfying witnesses of SyntheticCircuit(n) (ints) and their public signals."""
    from gosnark_b200.synthetic import SyntheticCircuit
    cs = [SyntheticCircuit(n, seed=0xBA7C0 + 977 * seed + p) for p in range(k)]
    return [c.witness for c in cs], [c.public_signals for c in cs]


def blindings(k, seed=0):
    return [((0x1234567 * (p + 3) + seed) << 180 | p) % R for p in range(k)], [((0x7654321 * (p + 5) + seed) << 170 | p) % R for p in range(k)]


def to_dev(arr):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def limbs(vals):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs(list(vals))


def split(words):
    """48 u64 (PiA | PiC | PiB) -> (PiA, PiB, PiC) Jacobian tuples."""
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    pa, pc = _unflatten_g1(words[:24])
    return pa, _unflatten_g2(words[24:48])[0], pc


def affine(p):
    pa, pb, pc = p
    return G1.affine(pa), G2.affine(pb), G1.affine(pc)


def expected(dlogs):
    a, b, c = dlogs
    return G1.affine(G1.mul_scalar(G1.G, a)), G2.affine(G2.mul_scalar(G2.G, b)), G1.affine(G1.mul_scalar(G1.G, c))


def words_of(p):
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
    pa, pb, pc = p
    return _flatten_g1([pa]), _flatten_g2([pb]), _flatten_g1([pc])


def batch_device(L, pk, r1cs, d_w, m, k, rs, ss, d_out, stream=None):
    return L.b200_groth16_prove_witness_batch_device(pk, r1cs, d_w.data_ptr(), m, k, _p(limbs(rs)), _p(limbs(ss)),
                                                     d_out.data_ptr(), None if stream is None else stream.cuda_stream)


def _p(a):
    from gosnark_b200._lib import ptr
    return ptr(a)


def batch_host(L, pk, r1cs, w_limbs, m, rs, ss):
    """b200_groth16_prove_witness_batch -> list of (PiA, PiB, PiC)."""
    from gosnark_b200._lib import check
    k = len(rs)
    pa, pb, pc = np.zeros(12 * k, np.uint64), np.zeros(24 * k, np.uint64), np.zeros(12 * k, np.uint64)
    check(L.b200_groth16_prove_witness_batch(pk, r1cs, _p(w_limbs), m, k, _p(limbs(rs)), _p(limbs(ss)), _p(pa), _p(pb), _p(pc)))
    return [split(np.concatenate([pa[12 * p:12 * p + 12], pc[12 * p:12 * p + 12], pb[24 * p:24 * p + 24]])) for p in range(k)]


def run_device_batch(L, pk, r1cs, w_limbs, m, rs, ss, stream=None):
    import torch
    from gosnark_b200._lib import check
    k = len(rs)
    d_out = torch.full((48 * k,), -1, dtype=torch.int64, device="cuda")
    check(batch_device(L, pk, r1cs, to_dev(w_limbs), m, k, rs, ss, d_out, stream))
    torch.cuda.synchronize()
    raw = d_out.cpu().numpy().view(np.uint64)
    return [split(raw[48 * p:48 * p + 48]) for p in range(k)]


def single_device(L, pk, r1cs, w_limbs_one, m, r, s):
    import torch
    from gosnark_b200._lib import check
    d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
    check(L.b200_groth16_prove_witness_device(pk, r1cs, to_dev(w_limbs_one).data_ptr(), m, _p(limbs([r])), _p(limbs([s])),
                                              d_out.data_ptr(), None))
    torch.cuda.synchronize()
    return split(d_out.cpu().numpy().view(np.uint64))


def load_pk(L, syn, ctx=0, acc=0, t=0):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    try:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, ctx))
        check(L.b200_config(_lib.CFG_ACC_MODE, acc))
        check(L.b200_config(_lib.CFG_TABLE_WINDOWS, t))
        return syn.load_pk()
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))
        check(L.b200_config(_lib.CFG_ACC_MODE, 0))
        check(L.b200_config(_lib.CFG_TABLE_WINDOWS, 0))


def verify_with(syn, proof, public):
    """groth16.VerifyProof under syn's real Vk with the given public signals."""
    from gosnark_b200._lib import check, ints_to_limbs, lib, ptr
    ok = ctypes.c_int(0)
    pa, pb, pc = words_of(proof)
    pub = ints_to_limbs(public)
    check(lib().b200_groth16_verify(ptr(syn.ic), syn.npublic + 1, ptr(syn.alpha1), ptr(syn.beta2), ptr(syn.gamma2),
                                    ptr(syn.delta2), ptr(pa), ptr(pb), ptr(pc), ptr(pub), len(public), ctypes.byref(ok)))
    return bool(ok.value)


def check_batch(L, syn, pk, proofs, wits, pubs, rs, ss, single=True, satisfied=None):
    """The three checks of the module docstring (satisfied[p] False: only the single-path equality and a refusal)."""
    for p, got in enumerate(proofs):
        sat = satisfied is None or satisfied[p]
        if sat:
            assert affine(got) == expected(syn.expected_dlogs(wits[p], rs[p], ss[p])), p
        if single or not sat:
            ref = single_device(L, pk, syn.r1cs.handle, limbs(wits[p]), syn.m, rs[p], ss[p])
            assert affine(got) == affine(ref), p
        assert verify_with(syn, got, pubs[p]) == sat, p


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("n,acc,ks", [(1 << 6, 0, (1, 2, 5)), ((1 << 12) + 2, 1, (1, 2, 5)), ((1 << 12) + 2, 2, (1, 2, 5)),
                                      (1 << 16, 0, (1, 4))], ids=["64", "4098-affine", "4098-xyzz", "65536"])
def test_sizes_and_entries(L, n, acc, ks):
    """Both entries, the device one on the library stream and on a torch side stream; k = 1 equals the single entry."""
    import torch
    from gosnark_b200._lib import check
    syn = circuit(n)
    pk = load_pk(L, syn, acc=acc)
    try:
        for k in ks:
            wits, pubs = witnesses(n, k, seed=k)
            rs, ss = blindings(k, seed=k)
            wl = limbs([v for w in wits for v in w])
            runs = {"host": batch_host(L, pk, syn.r1cs.handle, wl, syn.m, rs, ss),
                    "device": run_device_batch(L, pk, syn.r1cs.handle, wl, syn.m, rs, ss),
                    "device-side-stream": run_device_batch(L, pk, syn.r1cs.handle, wl, syn.m, rs, ss, torch.cuda.Stream())}
            check_batch(L, syn, pk, runs["device"], wits, pubs, rs, ss)
            for name in ("host", "device-side-stream"):
                assert [affine(p) for p in runs[name]] == [affine(p) for p in runs["device"]], (name, k)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("n", [1 << 6, 1 << 10])
def test_large_k(L, n):
    from gosnark_b200._lib import check
    syn = circuit(n)
    pk = load_pk(L, syn)
    try:
        for k in (33, 100):
            wits, pubs = witnesses(n, k, seed=k)
            rs, ss = blindings(k, seed=k)
            got = run_device_batch(L, pk, syn.r1cs.handle, limbs([v for w in wits for v in w]), syn.m, rs, ss)
            check_batch(L, syn, pk, got, wits, pubs, rs, ss, single=False)
            for p in (0, k // 2, k - 1):
                ref = single_device(L, pk, syn.r1cs.handle, limbs(wits[p]), syn.m, rs[p], ss[p])
                assert affine(got[p]) == affine(ref), p
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [1 << 6, (1 << 12) + 2])
def test_mixed_and_repeated_witnesses(L, n):
    """Satisfied witnesses next to unsatisfied ones (one signal off, which breaks the rows that read it; every entry
    random): each unsatisfied proof equals the single path's and is refused, its neighbours verify.  A repeated witness
    with other (r, s) and an identical triple twice give their own proofs."""
    import random
    from gosnark_b200._lib import check
    syn = circuit(n)
    pk = load_pk(L, syn)
    try:
        wits, pubs = witnesses(n, 4, seed=n)
        one_off = list(wits[1])
        one_off[n // 2 + 2] = (one_off[n // 2 + 2] + 1) % R
        rng = random.Random(n)
        every = [1] + [rng.randrange(R) for _ in range(syn.m - 1)]
        batch = [wits[0], one_off, wits[1], every, wits[2], wits[2], wits[3], wits[3]]
        bp = [pubs[0], pubs[1], pubs[1], [every[1]], pubs[2], pubs[2], pubs[3], pubs[3]]
        sat = [True, False, True, False, True, True, True, True]
        rs, ss = blindings(8, seed=n)
        rs[7], ss[7] = rs[6], ss[6]                 # an identical triple twice
        got = run_device_batch(L, pk, syn.r1cs.handle, limbs([v for w in batch for v in w]), syn.m, rs, ss)
        check_batch(L, syn, pk, got, batch, bp, rs, ss, satisfied=sat)
        assert affine(got[6]) == affine(got[7])
        assert affine(got[4]) != affine(got[5])
    finally:
        check(L.b200_pk_free(pk))


def row_values(csr, w):
    """(M w)_j for every row j of a CSR matrix (rowptr, col, val ints): a repeated (row, column) entry adds."""
    rowptr, col, val = csr
    return [sum(val[x] * w[int(col[x])] for x in range(int(rowptr[j]), int(rowptr[j + 1]))) % R for j in range(len(rowptr) - 1)]


class IrregularGroth16:
    """A seeded sparse R1CS over m signals [one, pub, x_0 ..] with n constraints, satisfiable by construction, and the CRS
    of groth16.GenerateTrustedSetup for it (Z = prod_{i=1..m-2} (x - i), so m = n + 3 gives len(Z) = n + 2):
      - A and B rows with 0 .. 3 terms, some empty; one A row and one B row of up to 512 terms;
      - explicit 0 and r - 1 coefficients; a repeated (row, column) entry in A, B and C (it acts as the sum);
      - every C row holds `one` and one column k with coefficient (a_j b_j - rest_j) / w_k, so that row j holds;
      - the last five private columns are used by no matrix.
    The CRS scalars come from the device's A^T l(T) (b200_qap_eval_at) with seeded toxic values."""

    def __init__(self, n, m, seed):
        import random
        from gosnark_b200._lib import check, ints_to_limbs, lib, limbs_to_ints, ptr
        from gosnark_b200.r1csqap import SparseR1CS
        from gosnark_b200.synthetic import mint_points
        rng = random.Random(seed)
        self.n, self.m, self.npublic = n, m, 1
        used = list(range(2, m - 5))
        pool_ab, pool_c = used + [0, 1], used + [1]
        w = [1, rng.randrange(1, R)] + [rng.randrange(1, R) for _ in range(m - 2)]
        coef = lambda: rng.choice([0, R - 1, 1, 2, rng.randrange(R), rng.randrange(R)])
        rows = {"A": [], "B": [], "C": []}
        for j in range(n):
            for M, dense, empty in (("A", n // 2, 3), ("B", n // 3, 5)):
                if j == dense:
                    cols = rng.sample(used, min(512, len(used)))
                elif j % 7 == empty:
                    cols = []
                else:
                    cols = [rng.choice(pool_ab) for _ in range(rng.randrange(1, 4))]
                rows[M].append([(c, coef()) for c in cols])
        if rows["A"][1]:
            rows["A"][1].append((rows["A"][1][0][0], 5))
        if rows["B"][2]:
            rows["B"][2].append((rows["B"][2][0][0], R - 3))
        csr = [self._csr(rows["A"]), self._csr(rows["B"])]
        a, b = row_values(csr[0], w), row_values(csr[1], w)
        for j in range(n):
            row = [(0, coef())] + [(rng.choice(pool_c), coef()) for _ in range(rng.randrange(0, 3))]
            if j == 4:
                row.append(row[0])
            k = used[(j * 7919) % len(used)]
            rest = sum(v * w[c] for c, v in row) % R
            row.append((k, (a[j] * b[j] - rest) * pow(w[k], -1, R) % R))
            rng.shuffle(row)
            rows["C"].append(row)
        csr.append(self._csr(rows["C"]))
        assert row_values(csr[2], w) == [x * y % R for x, y in zip(a, b)]
        self.witness, self.public_signals = w, [w[1]]
        self.r1cs = SparseR1CS(n, m, csr)
        self.toxic = dict(zip(("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta"), (rng.randrange(n + 1, R) for _ in range(5))))
        t, ka, kb, kg, kd = (self.toxic[k] for k in ("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta"))
        at_l, bt_l, ct_l, _ = self.r1cs.EvalAt(t)
        self.at_s, self.bt_s, self.ct_s = (limbs_to_ints(x) for x in (at_l, bt_l, ct_l))
        nz = m - 2
        self.z = np.zeros((nz + 1, 4), dtype=np.uint64)
        check(lib().b200_zero_poly(nz, ptr(self.z)))
        zt = 1
        for i in range(1, nz + 1):
            zt = zt * (t - i) % R
        l1 = self.npublic + 1
        inv_d, inv_g = pow(kd, -1, R), pow(kg, -1, R)
        lin = [(self.at_s[i] * kb + self.bt_s[i] * ka + self.ct_s[i]) % R for i in range(m)]
        self.kc = [0] * l1 + [inv_d * lin[i] % R for i in range(l1, m)]
        ptd = [zt * inv_d % R * pow(t, i, R) % R for i in range(m - 1)]
        self.at, self.b1, self.cd, self.ptd = (mint_points(1, ints_to_limbs(v)) for v in (self.at_s, self.bt_s, self.kc, ptd))
        self.b2 = mint_points(2, ints_to_limbs(self.bt_s))
        self.alpha1, self.beta1, self.delta1 = (mint_points(1, ints_to_limbs([v])) for v in (ka, kb, kd))
        self.beta2, self.delta2 = (mint_points(2, ints_to_limbs([v])) for v in (kb, kd))

    @staticmethod
    def _csr(rows):
        rowptr = np.zeros(len(rows) + 1, dtype=np.uint32)
        rowptr[1:] = np.cumsum([len(r) for r in rows])
        return rowptr, np.array([c for r in rows for c, _ in r], dtype=np.uint32), [v for r in rows for _, v in r]

    def load_pk(self):
        from gosnark_b200 import _lib
        from gosnark_b200._lib import check, lib, ptr
        h = _lib._h(0)
        check(lib().b200_groth16_pk_load(
            ptr(self.at), ptr(self.b1), ptr(self.b2), ptr(self.cd), self.m, ptr(self.ptd), self.m - 1, ptr(self.z),
            self.z.shape[0], ptr(self.alpha1), ptr(self.beta1), ptr(self.delta1), ptr(self.beta2), ptr(self.delta2),
            self.npublic, 0, h))
        return h.value

    def satisfied_dlogs(self, r, s):
        """Discrete logs of the proof of the satisfying witness when len(Z) = n + 1: then h(T) Z(T) = A(T) B(T) - C(T)."""
        w = self.witness
        t, ka, kb, kd = (self.toxic[k] for k in ("T", "Kalpha", "Kbeta", "Kdelta"))
        A, B, C = (sum(x * y for x, y in zip(v, w)) % R for v in (self.at_s, self.bt_s, self.ct_s))
        a, b = (A + ka + r * kd) % R, (B + kb + s * kd) % R
        c_msm = sum(x * y for x, y in zip(self.kc, w)) % R
        return a, b, (c_msm + (A * B - C) * pow(kd, -1, R) + s * a + r * b - r * s * kd) % R


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("n,m", [((1 << 12) + 2, (1 << 12) + 4), (300, 303)], ids=["4098", "300-m=n+3"])
def test_irregular_r1cs(L, n, m):
    """An irregular R1CS (IrregularGroth16): a batch of its satisfying witness, an unsatisfied one (x_0 + 1) and a random
    one equals the single path proof by proof; with len(Z) = n + 1 the satisfying witness's proof is also its known-dlog
    proof.  m = n + 3 gives len(Z) = n + 2: the px-and-division branch, looped per witness."""
    import random
    from gosnark_b200._lib import check
    inst = IrregularGroth16(n, m, seed=n ^ 0x5A5A)
    pk = inst.load_pk()
    try:
        w0 = inst.witness
        w1 = list(w0)
        w1[2] = (w1[2] + 1) % R
        rng = random.Random(m)
        w2 = [1] + [rng.randrange(R) for _ in range(m - 1)]
        batch = [w0, w1, w2, w0]
        rs, ss = blindings(4, seed=m)
        got = run_device_batch(L, pk, inst.r1cs.handle, limbs([v for w in batch for v in w]), m, rs, ss)
        for p, w in enumerate(batch):
            ref = single_device(L, pk, inst.r1cs.handle, limbs(w), m, rs[p], ss[p])
            assert affine(got[p]) == affine(ref), p
        if m == n + 2:
            assert affine(got[0]) == expected(inst.satisfied_dlogs(rs[0], ss[0]))
    finally:
        check(L.b200_pk_free(pk))
        inst.r1cs.free()


def _golden(golden_dir, name):
    with open(os.path.join(golden_dir, f"gobin_{name}.json")) as f:
        return json.load(f)


def groth_pk(setup):
    t3 = tuple
    g2t = lambda p: tuple(tuple(c) for c in p)
    pk = setup["Pk"]
    return {"Z": pk["Z"], "BACDelta": [t3(p) for p in pk["BACDelta"]], "PowersTauDelta": [t3(p) for p in pk["PowersTauDelta"]],
            "G1": {"Alpha": t3(pk["G1"]["Alpha"]), "Beta": t3(pk["G1"]["Beta"]), "Delta": t3(pk["G1"]["Delta"]),
                   "At": [t3(p) for p in pk["G1"]["At"]], "BACGamma": [t3(p) for p in pk["G1"]["BACGamma"]]},
            "G2": {"Beta": g2t(pk["G2"]["Beta"]), "Delta": g2t(pk["G2"]["Delta"]),
                   "BACGamma": [g2t(p) for p in pk["G2"]["BACGamma"]]}}


def groth_vk(setup):
    vk = setup["Vk"]
    g2t = lambda p: tuple(tuple(c) for c in p)
    return {"IC": [tuple(p) for p in vk["IC"]], "G1": {"Alpha": tuple(vk["G1"]["Alpha"])},
            "G2": {k: g2t(vk["G2"][k]) for k in ("Beta", "Gamma", "Delta")}}


@pytest.mark.parametrize("name", ["x3x5", "chain21", "mul"])
def test_golden_circuits(L, golden_dir, name):
    """The Go binary's circuits, the golden witness in a batch of three with other (r, s): each proof equals
    b200_groth16_prove with the golden px for its (r, s) and verifies under the golden Vk.  x3x5 and chain21 (len(Z) = n)
    take the short-Z quotient, mul the h-direct one."""
    from gosnark_b200 import groth16
    from gosnark_b200._lib import ints_to_limbs
    from gosnark_b200.bn128 import reduce_scalar
    from gosnark_b200.r1csqap import SparseR1CS
    g = _golden(golden_dir, name)
    cc = g["compiledcircuit"]
    a, b, c = cc["R1CS"]["A"], cc["R1CS"]["B"], cc["R1CS"]["C"]
    n, m = len(a), len(a[0])
    sp = SparseR1CS(n, m, (a, b, c))
    assert (len(g["groth16_setup"]["Pk"]["Z"]) == n + 1) == (name == "mul")
    dpk = groth16.DeviceProvingKey(groth_pk(g["groth16_setup"]), m, cc["NPublic"])
    try:
        w = ints_to_limbs([reduce_scalar(x) for x in g["witness"]])
        px = ints_to_limbs([int(x) % R for x in g["px"]])
        rs_ = [(0x1234567890ABCDEF << 100) + 17 * p for p in range(3)]
        ss_ = [(0xFEDCBA0987654321 << 90) + 29 * p for p in range(3)]
        got = dpk.prove_witness_batch_limbs(sp, np.concatenate([w] * 3), list(zip(rs_, ss_)))
        for p in range(3):
            ref = dpk.prove_limbs(w, px, rs_[p], ss_[p])
            for kk, G in (("PiA", G1), ("PiB", G2), ("PiC", G1)):
                assert G.affine(got[p][kk]) == G.affine(ref[kk]), (p, kk)
            assert groth16.VerifyProof(groth_vk(g["groth16_setup"]), got[p], g["public"])
    finally:
        dpk.free()
        sp.free()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("t", [1, 3])
def test_reduced_table_keys(L, t):
    """Keys with t stored window rows (B200_CFG_TABLE_WINDOWS): the batched sorts run over window groups."""
    from gosnark_b200._lib import check
    n = (1 << 12) + 2
    syn = circuit(n)
    pk = load_pk(L, syn, t=t)
    try:
        wits, pubs = witnesses(n, 3, seed=t)
        rs, ss = blindings(3, seed=t)
        got = run_device_batch(L, pk, syn.r1cs.handle, limbs([v for w in wits for v in w]), syn.m, rs, ss)
        check_batch(L, syn, pk, got, wits, pubs, rs, ss)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_two_contexts_in_flight_share_one_r1cs(L):
    """Batches on a context-0 and a context-1 key sharing one R1CS handle, on two streams, interleaved with single
    proofs on the same keys and streams, with no host synchronisation after the first call per context."""
    import torch
    from gosnark_b200._lib import check
    n = 1 << 12
    syn = circuit(n)
    pks = [load_pk(L, syn, ctx=c) for c in range(2)]
    try:
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        k = 3
        wits, pubs = witnesses(n, 2 * k, seed=77)
        d_w = [to_dev(limbs([v for w in wits[c * k:(c + 1) * k] for v in w])) for c in range(2)]
        d_one = [to_dev(limbs(wits[c])) for c in range(2)]
        rounds = 3
        outs, singles, blind = {}, {}, {}
        for c in range(2):      # the first call per (R1CS, context) builds its workspace and may synchronise
            rs, ss = blindings(k, seed=1000 + c)
            d = torch.zeros(48 * k, dtype=torch.int64, device="cuda")
            check(batch_device(L, pks[c], syn.r1cs.handle, d_w[c], syn.m, k, rs, ss, d, streams[c]))
        torch.cuda.synchronize()
        for j in range(rounds):
            for c in range(2):
                rs, ss = blindings(k, seed=10 * j + c)
                blind[(j, c)] = (rs, ss)
                outs[(j, c)] = torch.zeros(48 * k, dtype=torch.int64, device="cuda")
                check(batch_device(L, pks[c], syn.r1cs.handle, d_w[c], syn.m, k, rs, ss, outs[(j, c)], streams[c]))
                singles[(j, c)] = torch.zeros(48, dtype=torch.int64, device="cuda")
                check(L.b200_groth16_prove_witness_device(pks[c], syn.r1cs.handle, d_one[c].data_ptr(), syn.m, _p(limbs([rs[0]])),
                                                          _p(limbs([ss[0]])), singles[(j, c)].data_ptr(), streams[c].cuda_stream))
        torch.cuda.synchronize()
        for (j, c), d in outs.items():
            rs, ss = blind[(j, c)]
            raw = d.cpu().numpy().view(np.uint64)
            for p in range(k):
                w = wits[c * k + p]
                assert affine(split(raw[48 * p:48 * p + 48])) == expected(syn.expected_dlogs(w, rs[p], ss[p])), (j, c, p)
            assert affine(split(singles[(j, c)].cpu().numpy().view(np.uint64))) == expected(syn.expected_dlogs(wits[c], rs[0], ss[0]))
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_two_host_threads(L):
    """b200_groth16_prove_witness_batch from two host threads, thread c on the context-c key, one R1CS handle."""
    from gosnark_b200._lib import check
    n = 1 << 11
    syn = circuit(n)
    pks = [load_pk(L, syn, ctx=c) for c in range(2)]
    k, rounds = 4, 3
    wits, pubs = witnesses(n, 2 * k, seed=91)
    results, errs = {}, []

    def worker(c):
        try:
            wl = limbs([v for w in wits[c * k:(c + 1) * k] for v in w])
            for j in range(rounds):
                rs, ss = blindings(k, seed=100 * j + c)
                results[(c, j)] = (rs, ss, batch_host(L, pks[c], syn.r1cs.handle, wl, syn.m, rs, ss))
        except Exception as e:   # noqa: BLE001 - reported below
            errs.append(e)

    try:
        ths = [threading.Thread(target=worker, args=(c,)) for c in range(2)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        assert not errs, errs
        for (c, j), (rs, ss, proofs) in results.items():
            for p, got in enumerate(proofs):
                assert affine(got) == expected(syn.expected_dlogs(wits[c * k + p], rs[p], ss[p])), (c, j, p)
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


def pk_bytes(L, pk):
    from gosnark_b200._lib import check
    v = ctypes.c_size_t(0)
    check(L.b200_pk_device_bytes(pk, ctypes.byref(v)))
    return v.value


@pytest.mark.timeout(900)
def test_scratch_regrowth_without_host_sync(L):
    """k = 2, 8, 3, 8 on one stream with no host synchronisation between the calls: b200_pk_device_bytes grows at the
    first call and at the first k = 8, then stays; every proof is right."""
    import torch
    from gosnark_b200._lib import check
    n = 1 << 10
    syn = circuit(n)
    pk = load_pk(L, syn)
    try:
        st = torch.cuda.Stream()
        wits, pubs = witnesses(n, 8, seed=5)
        d_w = to_dev(limbs([v for w in wits for v in w]))
        sizes, outs = [pk_bytes(L, pk)], []
        for i, k in enumerate((2, 8, 3, 8)):
            rs, ss = blindings(k, seed=i)
            d = torch.zeros(48 * k, dtype=torch.int64, device="cuda")
            check(batch_device(L, pk, syn.r1cs.handle, d_w, syn.m, k, rs, ss, d, st))
            outs.append((k, rs, ss, d))
            sizes.append(pk_bytes(L, pk))
        assert sizes[0] < sizes[1] < sizes[2] == sizes[3] == sizes[4], sizes
        torch.cuda.synchronize()
        for k, rs, ss, d in outs:
            raw = d.cpu().numpy().view(np.uint64)
            for p in range(k):
                assert affine(split(raw[48 * p:48 * p + 48])) == expected(syn.expected_dlogs(wits[p], rs[p], ss[p])), (k, p)
    finally:
        check(L.b200_pk_free(pk))


def pick_window_bits(n):
    """capi.cu's pick_window_bits, restated: the window of a key's base set of n terms."""
    best, best_cost = 8, None
    for c in range(8, 19):
        cost = ((255 + c - 1) // c) * n * 10.0 + 2.0 * (1 << (c - 1)) * 14.0 * 4.0
        if best_cost is None or cost < best_cost:
            best, best_cost = c, cost
    return best


def msm_extras(k, c):
    """b200_msm_device_batch's documented extras at one window group: one launch once k * 2^(c-1) + 1 counters exceed
    64 Ki (multi-block scan), tail chunks (none below 65536 rows)."""
    return int(k * (1 << (c - 1)) + 1 > 65536) - int((1 << (c - 1)) + 1 > 65536)


def _launches(L, fn):
    from gosnark_b200._lib import check
    out = (ctypes.c_double * 8)()
    check(L.b200_profile_read(out))
    fn()
    check(L.b200_profile_read(out))
    return int(out[6])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [(1 << 12) + 2, 1 << 16])
def test_launch_count_does_not_grow_with_k(L, n):
    """From b200_profile_read: a batch of k issues the launches of a batch of one plus the batched MSM's extras of its
    two sorts (A/B1/B2 over m + 3 terms, C||PTD over 2m - 2), and fewer than k single proofs."""
    import torch
    from gosnark_b200._lib import check
    syn = circuit(n)
    pk = load_pk(L, syn)
    try:
        wits, _ = witnesses(n, 33, seed=3)
        d_w = to_dev(limbs([v for w in wits for v in w]))
        d_out = torch.zeros(48 * 33, dtype=torch.int64, device="cuda")
        c_ab, c_ch = pick_window_bits(syn.m + 3), pick_window_bits(2 * syn.m - 2)

        def batch(k):
            rs, ss = blindings(k)
            check(batch_device(L, pk, syn.r1cs.handle, d_w, syn.m, k, rs, ss, d_out))
        for k in (1, 2, 8, 33):      # warm-up: scratch and domains
            batch(k)
        base = _launches(L, lambda: batch(1))
        single = _launches(L, lambda: check(L.b200_groth16_prove_witness_device(
            pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, _p(limbs([syn.r])), _p(limbs([syn.s])), d_out.data_ptr(), None)))
        for k in (2, 8, 33):
            got = _launches(L, lambda: batch(k))
            assert got == base + msm_extras(k, c_ab) + msm_extras(k, c_ch), (k, got, base)
            assert got < k * single, (k, got, single)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(600)
def test_errors(L):
    """Every B200_EINVAL / B200_ERANGE of the two entries; an ERANGE in proof p leaves the outputs untouched and the next
    batch is right; a size-limit EINVAL leaves b200_pk_device_bytes unchanged; a witness entry >= r on the device entry is
    read as 0 and reported by no call."""
    import torch
    from gosnark_b200._lib import check
    n = 1 << 6
    syn = circuit(n)
    pk = load_pk(L, syn)
    other = circuit(n + 1)
    shard = syn.load_pk(0, 2)
    h, m = syn.r1cs.handle, syn.m
    try:
        k = 3
        wits, pubs = witnesses(n, k, seed=9)
        wl = limbs([v for w in wits for v in w])
        d_w = to_dev(wl)
        d_out = torch.zeros(48 * k, dtype=torch.int64, device="cuda")
        rs, ss = blindings(k)
        rl, sl = limbs(rs), limbs(ss)
        bad_r = limbs([rs[0], R, rs[2]])
        dev = lambda *a: L.b200_groth16_prove_witness_batch_device(*a)
        D, O = d_w.data_ptr(), d_out.data_ptr()
        cases = {
            "k = 0": (pk, h, D, m, 0, _p(rl), _p(sl), O, EINVAL),
            "bad key": (0, h, D, m, k, _p(rl), _p(sl), O, EINVAL),
            "bad r1cs": (pk, 0xDEAD, D, m, k, _p(rl), _p(sl), O, EINVAL),
            "null witness": (pk, h, None, m, k, _p(rl), _p(sl), O, EINVAL),
            "null r": (pk, h, D, m, k, None, _p(sl), O, EINVAL),
            "null s": (pk, h, D, m, k, _p(rl), None, O, EINVAL),
            "null out": (pk, h, D, m, k, _p(rl), _p(sl), None, EINVAL),
            "nw != m": (pk, h, D, m - 1, k, _p(rl), _p(sl), O, EINVAL),
            "r1cs m != key m": (pk, other.r1cs.handle, D, m, k, _p(rl), _p(sl), O, EINVAL),
            "sharded key": (shard, h, D, m, k, _p(rl), _p(sl), O, EINVAL),
            "r_1 >= r": (pk, h, D, m, k, _p(bad_r), _p(sl), O, ERANGE),
            "s_1 >= r": (pk, h, D, m, k, _p(rl), _p(bad_r), O, ERANGE),
        }
        before = pk_bytes(L, pk)
        for what, (key, r1, dw, nw, kk, r_, s_, out, code) in cases.items():
            assert dev(key, r1, dw, nw, kk, r_, s_, out, None) == code, what
        # size limits: k * nwin * (terms) sort entries reaching 2^31 (checked before r and s are read)
        big_k = (1 << 31) // (((255 + 7) // 8) * (m + 3)) + 1
        assert dev(pk, h, D, m, big_k, _p(rl), _p(sl), O, None) == EINVAL
        assert b"2^31" in L.b200_last_error()
        assert pk_bytes(L, pk) == before
        pa, pb, pc = np.zeros(12 * k, np.uint64), np.zeros(24 * k, np.uint64), np.zeros(12 * k, np.uint64)
        host = lambda key, r1, w, nw, kk, r_, s_: L.b200_groth16_prove_witness_batch(key, r1, w, nw, kk, r_, s_, _p(pa), _p(pb), _p(pc))
        assert host(pk, h, _p(wl), m, 0, _p(rl), _p(sl)) == EINVAL
        assert host(pk, h, None, m, k, _p(rl), _p(sl)) == EINVAL
        assert host(shard, h, _p(wl), m, k, _p(rl), _p(sl)) == EINVAL
        assert host(pk, h, _p(wl), m, k, _p(bad_r), _p(sl)) == ERANGE
        # a witness entry >= r in proof 1: ERANGE, outputs untouched, the next batch right
        bad = wl.copy()
        bad[m + 5] = limbs([R])[0]
        pa[:] = 7
        assert host(pk, h, _p(bad), m, k, _p(rl), _p(sl)) == ERANGE
        assert (pa == 7).all() and (pb == 0).all() and (pc == 0).all()
        got = batch_host(L, pk, h, wl, m, rs, ss)
        check_batch(L, syn, pk, got, wits, pubs, rs, ss, single=False)
        # the device entry reads it as 0 and reports it nowhere: proof 1 is that of witness 1 with the entry zeroed
        check(dev(pk, h, to_dev(bad).data_ptr(), m, k, _p(rl), _p(sl), O, None))
        torch.cuda.synchronize()
        raw = d_out.cpu().numpy().view(np.uint64)
        zeroed = wl[m:2 * m].copy()
        zeroed[5] = 0
        assert affine(split(raw[48:96])) == affine(single_device(L, pk, h, zeroed, m, rs[1], ss[1]))
        assert affine(split(raw[48:96])) != affine(single_device(L, pk, h, wl[m:2 * m], m, rs[1], ss[1]))
        for p in (0, 2):
            assert affine(split(raw[48 * p:48 * p + 48])) == expected(syn.expected_dlogs(wits[p], rs[p], ss[p])), p
        got = batch_host(L, pk, h, wl, m, rs, ss)
        check_batch(L, syn, pk, got, wits, pubs, rs, ss, single=False)
    finally:
        check(L.b200_pk_free(pk))
        check(L.b200_pk_free(shard))


@pytest.mark.timeout(600)
def test_measurement_mode(L):
    """b200_profile(2) (every MSM of a proof on the caller's stream) gives the same proofs."""
    from gosnark_b200._lib import check
    n = (1 << 12) + 2
    syn = circuit(n)
    pk = load_pk(L, syn)
    try:
        wits, pubs = witnesses(n, 3, seed=21)
        rs, ss = blindings(3, seed=21)
        wl = limbs([v for w in wits for v in w])
        normal = run_device_batch(L, pk, syn.r1cs.handle, wl, syn.m, rs, ss)
        check(L.b200_profile(2))
        try:
            serial = run_device_batch(L, pk, syn.r1cs.handle, wl, syn.m, rs, ss)
        finally:
            check(L.b200_profile(0))
        assert [affine(p) for p in serial] == [affine(p) for p in normal]
        check_batch(L, syn, pk, serial, wits, pubs, rs, ss, single=False)
    finally:
        check(L.b200_pk_free(pk))
