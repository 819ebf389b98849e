"""GPU: an out-of-range witness is reported by the host-pointer proof that received it, and by no other call.

b200_groth16_prove, b200_groth16_prove_witness, b200_pinocchio_prove and b200_pinocchio_prove_record_device write input
errors to an error word of their own key and read it back after their proof, on the key's prove context.  So a witness
entry >= r returns B200_ERANGE from its own call, leaves nothing behind for the next proof on the key or for a library
call, and is never seen by a proof on another key that is in flight from another host thread (the Groth16 calls wait
with the library mutex released).  Every valid proof is compared with its known-discrete-log expectation."""
import threading

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
G1, G2 = o.BN.G1, o.BN.G2
R = o.R
OK, ERANGE = 0, -4
PIN_ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


_made = {}


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    yield _lib.lib()
    for syn in _made.values():
        syn.r1cs.free()
    _made.clear()


def instance(kind, n):
    """CircuitGroth16 / CircuitPinocchio of n constraints, minted once per module."""
    from gosnark_b200.synthetic import CircuitGroth16, CircuitPinocchio
    if (kind, n) not in _made:
        _made[(kind, n)] = CircuitGroth16(n=n) if kind == "groth16" else CircuitPinocchio(n)
    return _made[(kind, n)]


def load_pk(L, syn, ctx):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    check(L.b200_config(_lib.CFG_PK_CONTEXT, ctx))
    try:
        return syn.load_pk()
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))


def out_of_range(w):
    """A copy of the witness limbs with one private entry set to r."""
    from gosnark_b200._lib import ints_to_limbs
    bad = w.copy()
    bad[3] = ints_to_limbs([R])[0]
    return bad


def groth16_call(L, entry, pk, syn, w, r, s):
    """(return code, affine (PiA, PiB, PiC)) of one host-pointer Groth16 proof."""
    from gosnark_b200._lib import ints_to_limbs, ptr
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
    rr, ss = ints_to_limbs([r]), ints_to_limbs([s])
    if entry == "prove":
        rc = L.b200_groth16_prove(pk, ptr(w), w.shape[0], ptr(syn.px), syn.px.shape[0], ptr(rr), ptr(ss), ptr(pa), ptr(pb),
                                  ptr(pc))
    else:
        rc = L.b200_groth16_prove_witness(pk, syn.r1cs.handle, ptr(w), w.shape[0], ptr(rr), ptr(ss), ptr(pa), ptr(pb), ptr(pc))
    return rc, (G1.affine(_unflatten_g1(pa)[0]), G2.affine(_unflatten_g2(pb)[0]), G1.affine(_unflatten_g1(pc)[0]))


def groth16_expected(syn, r, s):
    a, b, c = syn.expected_dlogs(None, r, s)
    return G1.affine(G1.mul_scalar(G1.G, a)), G2.affine(G2.mul_scalar(G2.G, b)), G1.affine(G1.mul_scalar(G1.G, c))


def pinocchio_call(L, entry, pk, syn, w):
    """(return code, proof dict) of one host-pointer Pinocchio proof; the record entry is finished on one rank."""
    import torch
    from gosnark_b200._lib import ptr
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
    if entry == "pinocchio_prove":
        rc = L.b200_pinocchio_prove(pk, ptr(w), w.shape[0], ptr(syn.px), syn.px.shape[0], ptr(g1), ptr(pb))
    else:
        rec = torch.zeros(256, dtype=torch.int64, device="cuda")      # one 2 KB record
        torch.cuda.synchronize()
        rc = L.b200_pinocchio_prove_record_device(pk, ptr(w), w.shape[0], ptr(syn.px), syn.px.shape[0], rec.data_ptr())
        if rc == OK:
            assert L.b200_pinocchio_finalize_records(rec.data_ptr(), 1, ptr(g1), ptr(pb)) == OK
    proof = dict(zip(PIN_ORDER, _unflatten_g1(g1)))
    proof["PiB"] = _unflatten_g2(pb)[0]
    return rc, proof


def assert_pinocchio_known_dlogs(proof, dlogs):
    for k in PIN_ORDER:
        assert G1.affine(proof[k]) == G1.affine(G1.mul_scalar(G1.G, dlogs[k])), k
    assert G2.affine(proof["PiB"]) == G2.affine(G2.mul_scalar(G2.G, dlogs["PiB"])), "PiB"


def g1_msm_succeeds(L):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check, ptr
    from gosnark_b200.synthetic import mint_points, rand_limbs
    bases = _lib._h(0)
    check(L.b200_g1_bases_load(ptr(mint_points(1, rand_limbs(4, 77))), 4, 0, bases))
    out = np.zeros(12, np.uint64)
    try:
        return L.b200_g1_msm(bases.value, ptr(rand_limbs(4, 78)), 4, ptr(out)) == OK
    finally:
        check(L.b200_bases_free(bases.value))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("ctx", [0, 1])
@pytest.mark.parametrize("entry", ["prove", "prove_witness", "pinocchio_prove", "pinocchio_record"])
def test_out_of_range_witness_reported_by_its_own_call(L, entry, ctx):
    """A witness entry >= r returns B200_ERANGE; the next valid proof on the same key (loaded under prove context `ctx`)
    equals its known-discrete-log expectation, and a b200_g1_msm afterwards returns B200_OK."""
    from gosnark_b200._lib import check
    kind = "pinocchio" if entry.startswith("pinocchio") else "groth16"
    syn = instance(kind, 1 << 10)
    pk = load_pk(L, syn, ctx)
    try:
        if kind == "groth16":
            assert groth16_call(L, entry, pk, syn, out_of_range(syn.w), syn.r, syn.s)[0] == ERANGE
            rc, proof = groth16_call(L, entry, pk, syn, syn.w, syn.r, syn.s)
            assert rc == OK
            assert proof == groth16_expected(syn, syn.r, syn.s)
        else:
            assert pinocchio_call(L, entry, pk, syn, out_of_range(syn.w))[0] == ERANGE
            rc, proof = pinocchio_call(L, entry, pk, syn, syn.w)
            assert rc == OK
            assert_pinocchio_known_dlogs(proof, syn.expected_dlogs())
        assert g1_msm_succeeds(L)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("ctxs", [(0, 1), (0, 0)], ids=["contexts-0-1", "contexts-0-0"])
@pytest.mark.parametrize("entry", ["prove", "prove_witness"])
def test_two_host_threads_errors_stay_with_their_key(L, entry, ctxs):
    """Two host threads, three rounds each, on two keys of one 2^13-constraint circuit loaded under prove contexts
    `ctxs`.  Thread A's witness has an entry >= r, so every one of its calls returns B200_ERANGE; thread B's proofs are
    valid, so every one of its calls succeeds and equals its own expectation.  The Groth16 host-pointer calls wait with
    the library mutex released, so the two threads' proofs are in flight together."""
    from gosnark_b200._lib import check
    syn = instance("groth16", 1 << 13)
    pks = [load_pk(L, syn, c) for c in ctxs]
    bad = out_of_range(syn.w)
    rounds = 3
    codes, proofs, errs = [], {}, []

    def worker_a():
        try:
            for _ in range(rounds):
                codes.append(groth16_call(L, entry, pks[0], syn, bad, syn.r, syn.s)[0])
        except Exception as e:   # noqa: BLE001 - reported below
            errs.append(e)

    def worker_b():
        try:
            for j in range(rounds):
                r_, s_ = (syn.r + 101 * j) % R, (syn.s + 103 * j) % R
                proofs[j] = (r_, s_, *groth16_call(L, entry, pks[1], syn, syn.w, r_, s_))
        except Exception as e:   # noqa: BLE001 - reported below
            errs.append(e)

    try:
        ths = [threading.Thread(target=worker_a), threading.Thread(target=worker_b)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        assert not errs, errs
        assert codes == [ERANGE] * rounds, codes
        assert sorted(proofs) == list(range(rounds))
        for j, (r_, s_, rc, proof) in proofs.items():
            assert rc == OK, (j, rc)
            assert proof == groth16_expected(syn, r_, s_), j
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))
