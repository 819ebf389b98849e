"""GPU: real proofs of satisfying witnesses that are almost entirely zero.

SyntheticCircuit(n) is the chain (x_0 + 5) x_0 = x_1, x_k x_(k-1) = x_(k+1), x_(n-1) x_(n-2) = pub; its R1CS does not
depend on x_0, so every x_0 gives a satisfying witness of the same key:
  x_0 = 0      w = [1, 0, 0, ...]:          B.w = 0 (and A.w = 5 in row 0 only), px = 0, h = 0;
  x_0 = r - 5  w = [1, 0, r - 5, 0, ...]:   A.w = 0 and C.w = 0, px = 0, h = 0;
  x_0 = r - 1  small values -4, 4, -16, -64, ... at the start of the chain, then full-width ones.
With h = 0 the quotient MSM of Groth16 carries only the blinding term, the A / B1 / B2 MSMs share a sort whose buckets are
nearly all empty, and the QAP front end interpolates zero vectors.  Every proof element must still be the exact k*G of the
QAP identity in the exponent (CircuitGroth16 / CircuitPinocchio.expected_dlogs) and verify under the real Vk with the
witness's own public signal (0 for the first two)."""
import ctypes

import numpy as np
import pytest

from oracle import ref_py as o

G1, G2 = o.BN.G1, o.BN.G2
R = o.R
X0 = {"zero": 0, "r-5": R - 5, "r-1": R - 1}
SIZES = [1 << 16, (1 << 12) + 2]
EINVAL = -3


def chain_witness(n, x0):
    """[one, pub, x_0 .. x_(n-1)] of SyntheticCircuit(n) from x_0."""
    xs = [x0 % R, (x0 + 5) * x0 % R]
    for k in range(1, n - 1):
        xs.append(xs[k] * xs[k - 1] % R)
    return [1, xs[n - 1] * xs[n - 2] % R] + xs[:n]


def test_chain_witness_shapes():
    """The witnesses are what the module docstring says, and satisfy every row (runs without a GPU)."""
    n = 40
    assert chain_witness(n, 0) == [1] + [0] * (n + 1)
    assert chain_witness(n, R - 5) == [1, 0, R - 5] + [0] * (n - 1)
    w = chain_witness(n, R - 1)
    assert w[2:8] == [R - 1, R - 4, 4, R - 16, R - 64, 1024]
    # A.w, B.w and C.w row by row: (x_0 + 5) x_0 = x_1, x_k x_(k-1) = x_(k+1), x_(n-1) x_(n-2) = pub
    for x0 in X0.values():
        w = chain_witness(n, x0)
        xs, pub = w[2:], w[1]
        assert (xs[0] + 5) * xs[0] % R == xs[1]
        assert all(xs[k] * xs[k - 1] % R == (xs[k + 1] if k + 1 < n else pub) for k in range(1, n))


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


_made = {}


def instance(protocol, n):
    """CircuitGroth16 / CircuitPinocchio of n constraints, minted once per module."""
    from gosnark_b200.synthetic import CircuitGroth16, CircuitPinocchio
    if (protocol, n) not in _made:
        _made[(protocol, n)] = CircuitGroth16(n=n) if protocol == "groth16" else CircuitPinocchio(n)
    return _made[(protocol, n)]


@pytest.fixture(scope="module")
def _free_instances():
    yield
    for syn in _made.values():
        syn.r1cs.free()
    _made.clear()


def load_pk(L, syn, mode):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    check(L.b200_config(_lib.CFG_ACC_MODE, mode))
    try:
        return syn.load_pk()
    finally:
        check(L.b200_config(_lib.CFG_ACC_MODE, _lib.ACC_AUTO))


def limbs(v):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs([v])


def split(words):
    """48 u64 (PiA | PiC | PiB) -> (PiA, PiB, PiC)."""
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    pa, pc = _unflatten_g1(words[:24])
    return pa, _unflatten_g2(words[24:48])[0], pc


def groth16_verify(L, syn, proof, public):
    """groth16.VerifyProof on the GPU under the instance's real Vk with the given public signals."""
    from gosnark_b200._lib import check, ptr
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
    pa, pb, pc = proof
    ok = ctypes.c_int(0)
    check(L.b200_groth16_verify(ptr(syn.ic), syn.npublic + 1, ptr(syn.alpha1), ptr(syn.beta2), ptr(syn.gamma2),
                                ptr(syn.delta2), ptr(_flatten_g1([pa])), ptr(_flatten_g2([pb])), ptr(_flatten_g1([pc])),
                                ptr(limbs(public[0])), 1, ctypes.byref(ok)))
    return bool(ok.value)


def check_groth16_entry_points(L, syn, pk, w_ints, px, name, host_witness=True):
    """Prove w_ints with (r, s) of the instance through b200_groth16_prove (px), b200_groth16_prove_witness (unless
    host_witness is False) and b200_groth16_prove_witness_device on a side stream; every proof must be the
    known-discrete-log proof, and it verifies with the witness's public signal and not with another."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    w = ints_to_limbs(w_ints)
    a, b, c = syn.expected_dlogs(witness=w_ints, r=syn.r, s=syn.s)
    exp = (G1.affine(G1.mul_scalar(G1.G, a)), G2.affine(G2.mul_scalar(G2.G, b)), G1.affine(G1.mul_scalar(G1.G, c)))
    rr, ss = ptr(limbs(syn.r)), ptr(limbs(syn.s))
    got = {}
    pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
    check(L.b200_groth16_prove(pk, ptr(w), syn.m, ptr(px), px.shape[0], rr, ss, ptr(pa), ptr(pb), ptr(pc)))
    got["px"] = split(np.concatenate([pa, pc, pb]))
    if host_witness:
        pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
        check(L.b200_groth16_prove_witness(pk, syn.r1cs.handle, ptr(w), syn.m, rr, ss, ptr(pa), ptr(pb), ptr(pc)))
        got["witness"] = split(np.concatenate([pa, pc, pb]))
    d_w = torch.from_numpy(w.reshape(-1).view(np.int64)).cuda()
    d_out = torch.full((48,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    check(L.b200_groth16_prove_witness_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, rr, ss, d_out.data_ptr(),
                                              side.cuda_stream))
    side.synchronize()
    got["witness-device"] = split(d_out.cpu().numpy().view(np.uint64))
    for entry, (qa, qb, qc) in got.items():
        assert (G1.affine(qa), G2.affine(qb), G1.affine(qc)) == exp, (name, entry)
    assert groth16_verify(L, syn, got["witness-device"], [w_ints[1]]), name
    assert not groth16_verify(L, syn, got["witness-device"], [(w_ints[1] + 1) % R]), name


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("n", SIZES, ids=["65536", "4098"])
def test_groth16_degenerate_witnesses(L, _free_instances, n, mode):
    """b200_groth16_prove (px from the sparse front end), b200_groth16_prove_witness and
    b200_groth16_prove_witness_device under the batched-affine (1) and XYZZ (2) accumulation: for each x_0 every entry
    point returns the known-discrete-log proof, which verifies with the witness's public signal and fails with another."""
    from gosnark_b200._lib import check, ints_to_limbs
    syn = instance("groth16", n)
    pk = load_pk(L, syn, mode)
    try:
        for name, x0 in X0.items():
            w_ints = chain_witness(n, x0)
            px = syn.px_of(ints_to_limbs(w_ints))
            if name != "r-1":
                assert not px.any(), name                       # A.w * B.w - C.w = 0 on every row
                assert w_ints[1] == 0
            check_groth16_entry_points(L, syn, pk, w_ints, px, name)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_groth16_degenerate_witnesses_at_2_20(L, _free_instances):
    """The all-zero and the A.w = C.w = 0 witnesses at 2^20 constraints, the benchmark size, through the device witness
    entry (and px = 0 through b200_groth16_prove) at the automatic accumulation mode."""
    from gosnark_b200._lib import check, ints_to_limbs
    n = 1 << 20
    syn = instance("groth16", n)
    pk = syn.load_pk()
    try:
        for name in ("zero", "r-5"):
            w_ints = chain_witness(n, X0[name])
            px = syn.px_of(ints_to_limbs(w_ints))
            assert not px.any(), name
            check_groth16_entry_points(L, syn, pk, w_ints, px, name, host_witness=False)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("n", SIZES, ids=["65536", "4098"])
def test_pinocchio_degenerate_witnesses(L, _free_instances, n, mode):
    """b200_pinocchio_prove under both accumulations: for each x_0 all eight elements equal the known discrete logs and
    the proof verifies under the real Vk with the witness's public signal, except where PiB is the point at infinity,
    which the verifier's pairing rejects as the reference does."""
    from gosnark_b200._lib import B200Error, check, ints_to_limbs, ptr
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    syn = instance("pinocchio", n)
    order = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")
    pk = load_pk(L, syn, mode)
    try:
        for name, x0 in X0.items():
            w_ints = chain_witness(n, x0)
            w = ints_to_limbs(w_ints)
            px = syn.px_of(w)
            g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
            check(L.b200_pinocchio_prove(pk, ptr(w), syn.m, ptr(px), px.shape[0], ptr(g1), ptr(pb)))
            proof = dict(zip(order, _unflatten_g1(g1)))
            proof["PiB"] = _unflatten_g2(pb)[0]
            exp = syn.expected_dlogs(w_ints)
            if name != "r-1":
                assert exp["PiH"] == 0 and exp["PiC"] == 0, name
            for k in order:
                assert G1.affine(proof[k]) == G1.affine(G1.mul_scalar(G1.G, exp[k])), (name, k)
            assert G2.affine(proof["PiB"]) == G2.affine(G2.mul_scalar(G2.G, exp["PiB"])), (name, "PiB")
            if exp["PiB"] == 0:
                # x_0 = 0: B.w = 0, so PiB is the G2 point at infinity.  The reference's Pairing panics on it
                # (bn128.go:238-241), so its VerifyProof can never accept such a proof; here the pairing call refuses it.
                with pytest.raises(B200Error) as e:
                    syn.verify(proof, [w_ints[1]])
                assert e.value.code == EINVAL and "G2 point at infinity" in str(e.value), name
            else:
                assert syn.verify(proof, [w_ints[1]]), name
    finally:
        check(L.b200_pk_free(pk))
