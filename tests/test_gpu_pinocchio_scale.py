"""GPU: Pinocchio proving (snark.go:254-289) at benchmark sizes on a REAL key (synthetic.CircuitPinocchio: the key and Vk of
snark.GenerateTrustedSetup for seeded toxic values, every point k*G with a known k).  At these sizes the prove path takes
what the golden circuits (<= 21 constraints) never reach: the batched-affine accumulation tree with several slices per
bucket, the fused NTT passes of the division, one digit sort shared by the G2 set B and four G1 sets, bucket phases on
three side streams, the G1T MSM after a real division, and whole MSMs dealt to ranks.  Every proof element is compared
with k*G for its expected k, exactly, so one wrong addition anywhere fails."""
import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
G1, G2 = o.BN.G1, o.BN.G2
ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")
OTHER_WITNESS_SEED = 0x5EED0101


@pytest.fixture(scope="module")
def instance():
    """CircuitPinocchio(n), minted once per module (a key of 2^16 constraints takes a while to mint)."""
    from gosnark_b200 import _lib
    from gosnark_b200.synthetic import CircuitPinocchio
    _lib.init()
    made = {}

    def get(n):
        if n not in made:
            made[n] = CircuitPinocchio(n)
        return made[n]
    yield get
    for syn in made.values():
        syn.r1cs.free()


def load_pk(syn, mode, rank=0, world=1):
    """Proving key (shard rank / world) with the bucket accumulation forced to batched affine (1) or XYZZ (2)."""
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check, lib
    check(lib().b200_config(_lib.CFG_ACC_MODE, mode))
    try:
        return syn.load_pk(rank, world)
    finally:
        check(lib().b200_config(_lib.CFG_ACC_MODE, _lib.ACC_AUTO))


def proof_of(g1, pb):
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    proof = dict(zip(ORDER, _unflatten_g1(g1)))
    proof["PiB"] = _unflatten_g2(pb)[0]
    return proof


def prove(pk, w, px):
    from gosnark_b200._lib import check, lib, ptr
    g1, pb = np.zeros(84, dtype=np.uint64), np.zeros(24, dtype=np.uint64)
    check(lib().b200_pinocchio_prove(pk, ptr(w), w.shape[0], ptr(px), px.shape[0], ptr(g1), ptr(pb)))
    return proof_of(g1, pb)


def assert_known_dlogs(proof, dlogs):
    for k in ORDER:
        assert G1.affine(proof[k]) == G1.affine(G1.mul_scalar(G1.G, dlogs[k])), k
    assert G2.affine(proof["PiB"]) == G2.affine(G2.mul_scalar(G2.G, dlogs["PiB"])), "PiB"


def assert_same(p, q):
    for k in ORDER:
        assert G1.affine(p[k]) == G1.affine(q[k]), k
    assert G2.affine(p["PiB"]) == G2.affine(q["PiB"]), "PiB"


@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("n", [1 << 12, (1 << 12) + 2, 1 << 16])
def test_pinocchio_prove_known_dlogs_and_verifies(instance, n, mode):
    """b200_pinocchio_prove under the batched-affine (1) and XYZZ (2) accumulation: all eight elements equal k*G for the k
    of the QAP identity and the proof passes snark.VerifyProof against the real Vk; a second proof on the same key —
    another witness, so the sort scratch and the cached divisor inverse are reused — matches its own expectation and
    verifies, and a proof that mixes elements of the two is rejected.  n = 2^12 + 2 gives a quotient of 2^12 + 1
    coefficients: the division's transforms double to 2^14 points and the interpolation of px crosses a power of two.

    A wrong public input is NOT rejected, here as in the reference: VerifyProof binds public signals only through
    IC = A[0..NPublic] (snark.go:333-336), and SyntheticCircuit's public signal occurs only in C, so IC[1] is the point at
    infinity."""
    from gosnark_b200._lib import check, ints_to_limbs, lib
    from gosnark_b200.synthetic import SyntheticCircuit
    syn = instance(n)
    pk = load_pk(syn, mode)
    proof = prove(pk, syn.w, syn.px)
    assert_known_dlogs(proof, syn.expected_dlogs())
    assert syn.verify(proof)
    assert syn.k["IC"][1] == 0 and syn.verify(proof, [(syn.circuit.public_signals[0] + 1) % o.R])
    other = SyntheticCircuit(n, seed=OTHER_WITNESS_SEED)
    w2 = ints_to_limbs(other.witness)
    proof2 = prove(pk, w2, syn.px_of(w2))
    assert_known_dlogs(proof2, syn.expected_dlogs(other.witness))
    assert syn.verify(proof2, other.public_signals)
    assert not syn.verify(dict(proof, PiH=proof2["PiH"]))          # the QAP divisibility check fails
    check(lib().b200_pk_free(pk))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("world", [2, 3, 8])
def test_pinocchio_sharded_records_known_dlogs(instance, world):
    """Whole MSMs dealt to `world` ranks (b200_pinocchio_pk_load_shard, emulated on one GPU): every rank's 2 KB record from
    b200_pinocchio_prove_record_device, concatenated as the all-gather would and summed by b200_pinocchio_finalize_records,
    equals the single-GPU proof and the known discrete logs at 2^12 constraints (batched-affine accumulation)."""
    import torch
    from gosnark_b200._lib import check, lib, ptr
    syn = instance(1 << 12)
    L = lib()
    single = load_pk(syn, 1)
    pks = [load_pk(syn, 1, rk, world) for rk in range(world)]
    recs = torch.zeros(256 * world, dtype=torch.int64, device="cuda")      # world x 2 KB
    torch.cuda.synchronize()
    for rk, pk in enumerate(pks):
        check(L.b200_pinocchio_prove_record_device(pk, ptr(syn.w), syn.m, ptr(syn.px), syn.px.shape[0],
                                                   recs[256 * rk:].data_ptr()))
    g1, pb = np.zeros(84, dtype=np.uint64), np.zeros(24, dtype=np.uint64)
    check(L.b200_pinocchio_finalize_records(recs.data_ptr(), world, ptr(g1), ptr(pb)))
    sharded = proof_of(g1, pb)
    assert_known_dlogs(sharded, syn.expected_dlogs())
    assert_same(sharded, prove(single, syn.w, syn.px))
    for pk in pks + [single]:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(600)
def test_pinocchio_and_groth16_share_context_workspaces(instance):
    """Keys of different sizes and protocols on prove context 0 share its polynomial workspaces and NTT plans, which grow
    on demand: Pinocchio at 2^12, Pinocchio at 2^16, Groth16 at 2^14, then Pinocchio at 2^12 again (its divisor cache
    made before the workspaces grew) — each proof equals its own known-discrete-log expectation."""
    from gosnark_b200._lib import check, ints_to_limbs, lib, ptr
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    from gosnark_b200.synthetic import CircuitGroth16
    L = lib()
    small, large = instance(1 << 12), instance(1 << 16)
    groth = CircuitGroth16(14)
    pk_small, pk_large, pk_groth = small.load_pk(), large.load_pk(), groth.load_pk()

    def groth16_proof():
        pa, pb, pc = np.zeros(12, dtype=np.uint64), np.zeros(24, dtype=np.uint64), np.zeros(12, dtype=np.uint64)
        check(L.b200_groth16_prove(pk_groth, ptr(groth.w), groth.m, ptr(groth.px), groth.px.shape[0],
                                   ptr(ints_to_limbs([groth.r])), ptr(ints_to_limbs([groth.s])), ptr(pa), ptr(pb), ptr(pc)))
        ea, eb, ec = groth.expected_dlogs()
        assert G1.affine(_unflatten_g1(pa)[0]) == G1.affine(G1.mul_scalar(G1.G, ea))
        assert G2.affine(_unflatten_g2(pb)[0]) == G2.affine(G2.mul_scalar(G2.G, eb))
        assert G1.affine(_unflatten_g1(pc)[0]) == G1.affine(G1.mul_scalar(G1.G, ec))

    assert_known_dlogs(prove(pk_small, small.w, small.px), small.expected_dlogs())
    assert_known_dlogs(prove(pk_large, large.w, large.px), large.expected_dlogs())
    groth16_proof()
    assert_known_dlogs(prove(pk_small, small.w, small.px), small.expected_dlogs())
    for pk in (pk_small, pk_large, pk_groth):
        check(L.b200_pk_free(pk))
    groth.r1cs.free()


@pytest.mark.timeout(600)
def test_pinocchio_accumulation_modes_by_launch_count(instance, capsys):
    """b200_profile shows which accumulation a 2^12 Pinocchio proof ran: under the batched-affine tree (mode 1) each of
    its rounds is three launches, so the proof issues more kernel launches than under XYZZ (mode 2); in both, seven G1
    bucket phases (A, Ap, Bp, C, Cp, Kp, G1T) and one G2 phase (B) run."""
    import ctypes
    from gosnark_b200._lib import check, lib
    syn = instance(1 << 12)
    L = lib()
    prof = {}
    for mode in (1, 2):
        pk = load_pk(syn, mode)
        prove(pk, syn.w, syn.px)                  # first proof: NTT plans and the divisor inverse are built here
        out = (ctypes.c_double * 8)()
        check(L.b200_profile(1))
        try:
            check(L.b200_profile_read(out))       # reset the counters
            proof = prove(pk, syn.w, syn.px)
            check(L.b200_profile_read(out))
        finally:
            check(L.b200_profile(0))
        check(L.b200_pk_free(pk))
        assert_known_dlogs(proof, syn.expected_dlogs())
        prof[mode] = list(out)
        assert (out[1], out[4]) == (7, 1), (mode, prof[mode])
    with capsys.disabled():
        print(f"\n2^12 Pinocchio proof: kernel launches {prof[1][6]:.0f} (batched affine) vs {prof[2][6]:.0f} (XYZZ)")
    assert prof[1][6] > prof[2][6]
