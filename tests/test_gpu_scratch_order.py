"""GPU: library calls and context-0 proofs in flight share context 0's scratch (its R1csWork on an R1CS, its polynomial
workspace).  A proof enqueued on the caller's stream computes its quotient on the key's side stream 3, and the library
stream runs b200_qap_px / b200_poly_mul / b200_poly_div: each use of the scratch must wait for the previous one on the
device.  Each interleaving runs once, at 2^20 constraints, and both results are checked against references that do not
come from the GPU: the proof against its known discrete logs, px against the barycentric values of A w, B w, C w."""
import random
import threading

import numpy as np
import pytest

from fr_ref import R, check_qap_px, horner, rand_limbs, to_ints
from test_gpu_prove_witness import affine, expected, host_prove_witness, limbs, split, to_dev, witness_device

pytestmark = pytest.mark.gpu
N = 1 << 20


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


@pytest.fixture(scope="module")
def setup(L):
    """A context-0 key of CircuitGroth16(2^20) with its R1CS, a second satisfying witness, and one warm-up of each entry
    involved (domains, workspaces and the key's division cache exist, so the timed calls allocate nothing big)."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    from gosnark_b200.synthetic import CircuitGroth16, SyntheticCircuit
    syn = CircuitGroth16(n=N)
    pk = syn.load_pk()
    w2 = SyntheticCircuit(N, seed=0x5EED0777).witness
    d_w, d_px = to_dev(syn.w), to_dev(syn.px)
    out = torch.zeros(48, dtype=torch.int64, device="cuda")
    check(witness_device(L, pk, syn.r1cs.handle, d_w, syn.m, syn.r, syn.s, out))
    check(L.b200_groth16_prove_device(pk, d_w.data_ptr(), syn.m, d_px.data_ptr(), syn.px.shape[0], ptr(limbs(syn.r)),
                                      ptr(limbs(syn.s)), out.data_ptr(), None))
    torch.cuda.synchronize()
    syn.r1cs.combine_limbs(ints_to_limbs(w2))
    exp = expected(syn.expected_dlogs())
    assert affine(split(out.cpu().numpy().view(np.uint64))) == exp
    yield syn, pk, w2, d_w, d_px, exp
    check(L.b200_pk_free(pk))
    syn.r1cs.free()


def px_of_w2(syn, w2):
    from gosnark_b200._lib import ints_to_limbs
    return syn.r1cs.combine_limbs(ints_to_limbs(w2))


def check_px_w2(syn, w2, out):
    rng = random.Random(7)
    check_qap_px(syn.circuit.csr, w2, out, rng.randrange(N + 1, R), [1, N, rng.randrange(2, N)])


@pytest.mark.timeout(900)
def test_witness_proof_on_stream_then_qap_px(L, setup):
    """(a) b200_groth16_prove_witness_device on a torch stream, then at once b200_qap_px on the same R1CS handle from
    another witness: both front ends use context 0's R1csWork."""
    import torch
    from gosnark_b200._lib import check
    syn, pk, w2, d_w, _, exp = setup
    stream = torch.cuda.Stream()
    out = torch.full((48,), -1, dtype=torch.int64, device="cuda")
    check(witness_device(L, pk, syn.r1cs.handle, d_w, syn.m, syn.r, syn.s, out, stream))
    got_px = px_of_w2(syn, w2)
    torch.cuda.synchronize()
    assert affine(split(out.cpu().numpy().view(np.uint64))) == exp
    check_px_w2(syn, w2, got_px)


@pytest.mark.timeout(900)
def test_px_proof_on_stream_then_poly_mul_and_div(L, setup):
    """(b) b200_groth16_prove_device fed px on a torch stream divides with context 0's polynomial workspace on side stream
    3; at once b200_poly_mul, then in a second round b200_poly_div, use the same buffers on the library stream, at sizes
    that fit the grown buffers (no reallocation, so no implicit device synchronisation)."""
    import torch
    from gosnark_b200._lib import check, ptr
    syn, pk, _, d_w, d_px, exp = setup
    stream = torch.cuda.Stream()
    rr, ss = limbs(syn.r), limbs(syn.s)

    def prove(out):
        check(L.b200_groth16_prove_device(pk, d_w.data_ptr(), syn.m, d_px.data_ptr(), syn.px.shape[0], ptr(rr), ptr(ss),
                                          out.data_ptr(), stream.cuda_stream))

    # round 1: a * x^(nb-1) at lo = 2^21 - 1 (the proof's own transforms are 2^21 points)
    na, nb = 1 << 20, 1 << 20
    a = rand_limbs(na, 31)
    e = np.zeros((nb, 4), dtype=np.uint64)
    e[nb - 1, 0] = 1
    prod = np.zeros((na + nb - 1, 4), dtype=np.uint64)
    out = torch.full((48,), -1, dtype=torch.int64, device="cuda")
    prove(out)
    check(L.b200_poly_mul(ptr(a), na, ptr(e), nb, ptr(prod)))
    torch.cuda.synchronize()
    assert affine(split(out.cpu().numpy().view(np.uint64))) == exp
    assert not prod[: nb - 1].any() and np.array_equal(prod[nb - 1:], a)
    # round 2: a division with a quotient of 2^19 coefficients
    nq, nb = 1 << 19, 9
    a, b = rand_limbs(nq + nb - 1, 32), rand_limbs(nb, 33)
    b[nb - 1] = (1, 0, 0, 0)
    q, rem = np.zeros((nq, 4), dtype=np.uint64), np.zeros((nb - 1, 4), dtype=np.uint64)
    out = torch.full((48,), -1, dtype=torch.int64, device="cuda")
    prove(out)
    check(L.b200_poly_div(ptr(a), a.shape[0], ptr(b), nb, ptr(q), ptr(rem)))
    torch.cuda.synchronize()
    assert affine(split(out.cpu().numpy().view(np.uint64))) == exp
    t = random.Random(34).randrange(R)
    assert horner(to_ints(a), t) == (horner(to_ints(q), t) * horner(to_ints(b), t) + horner(to_ints(rem), t)) % R


@pytest.mark.timeout(900)
def test_two_threads_host_witness_proof_and_qap_px(L, setup):
    """(c) Two host threads: one proves with b200_groth16_prove_witness (host pointers; the wait runs with the library
    mutex released), the other calls b200_qap_px on the same R1CS from another witness."""
    syn, pk, w2, _, _, exp = setup
    res, errs = {}, []
    go = threading.Barrier(2)

    def run(key, fn):
        try:
            go.wait()
            res[key] = fn()
        except Exception as ex:      # re-raised below, in the test's thread
            errs.append(ex)

    threads = [threading.Thread(target=run, args=("proof", lambda: host_prove_witness(L, pk, syn.r1cs.handle, syn.w, syn.r, syn.s))),
               threading.Thread(target=run, args=("px", lambda: px_of_w2(syn, w2)))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errs:
        raise errs[0]
    assert affine(res["proof"]) == exp
    check_px_w2(syn, w2, res["px"])
