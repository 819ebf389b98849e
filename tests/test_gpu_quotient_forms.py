"""GPU: witness-fed proving when len(Z) is neither n + 1 nor n, so the quotient is px divided by the key's Z.

The IrregularR1CS of test_gpu_prove_unsatisfied.py with m = n + 3 signals has len(Z) = n + 2: every witness entry forms
px on the device and divides it by Z, one witness at a time, also inside a batch.  For Pinocchio (keys minted by
b200_pinocchio_setup_pk, whole and 3-way sharded) every witness entry must give the proof of b200_pinocchio_prove with
that witness's px.  For Groth16, the 8-way shard's batch records must finalise to the unsharded batch: at world 8 more
than one rank holds PowersTauDelta indices, so some rank's slice of the quotient starts past its first coefficient and
is copied out of the full quotient.  Satisfied and unsatisfied witnesses alike.

Proofs are compared as group elements (affine): the MSM's counting sort scatters a bucket's entries with atomics, so
the Jacobian words of one proof differ from run to run."""
import random

import numpy as np
import pytest

from oracle import ref_py as o
from test_gpu_prove_unsatisfied import L, IrregularGroth16, IrregularR1CS, satisfied  # noqa: F401  (L: fixture)

pytestmark = pytest.mark.gpu
R = o.R
G1, G2 = o.BN.G1, o.BN.G2
SIZES = [300, (1 << 12) - 5]


def limbs(vals):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs(list(vals))


def to_dev(arr):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def d_words(n_words):
    import torch
    t = torch.full((n_words,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    return t


def host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64).copy()


def witnesses(circ, seed):
    """The satisfying witness, one with x_0 off by one, and a random one (both unsatisfied)."""
    w_bad = list(circ.witness)
    w_bad[2] = (w_bad[2] + 1) % R
    rng = random.Random(seed)
    w_rand = [1] + [rng.randrange(R) for _ in range(circ.m - 1)]
    assert not satisfied(circ.csr, w_bad) and not satisfied(circ.csr, w_rand)
    return [list(circ.witness), w_bad, w_rand]


# ---- Pinocchio -----------------------------------------------------------------------------------------------------
def pin_affine(words):
    """108 u64 (seven G1 Jacobian points, then PiB) -> affine points."""
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    return [G1.affine(p) for p in _unflatten_g1(words[:84])] + [G2.affine(_unflatten_g2(words[84:108])[0])]


def pin_proofs(words, k):
    return [pin_affine(words[108 * p:108 * p + 108]) for p in range(k)]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("n", SIZES)
def test_pinocchio_px_division(L, n):
    """b200_pinocchio_prove_witness(_device), a mixed batch of 3 through b200_pinocchio_prove_witness_batch_device, and
    the batch records of a 3-way shard finalised by b200_pinocchio_finalize_records_batch_device all equal
    b200_pinocchio_prove with each witness's px."""
    from gosnark_b200 import snark
    from gosnark_b200._lib import check, ptr
    from gosnark_b200.r1csqap import SparseR1CS
    m = n + 3
    circ = IrregularR1CS(n, m, seed=n ^ 0x5A5A)
    sp = SparseR1CS(n, m, circ.csr)
    rng = random.Random(n)
    tox = {k: rng.randrange(n + 2, R) for k in snark.SparseSetup.TOXIC}
    keys = []
    try:
        whole = snark.GenerateTrustedSetupResident(sp, circ.npublic, toxic=tox)
        keys.append(whole.pk)
        shards = [snark.GenerateTrustedSetupResident(sp, circ.npublic, toxic=tox, rank=g, world=3) for g in range(3)]
        keys += [s.pk for s in shards]
        wits = witnesses(circ, seed=n)
        wl = [limbs(w) for w in wits]
        ref = []
        for w in wl:
            px = sp.combine_limbs(w, want_abc=False)[3]
            p = whole.pk.prove_limbs(w, px)
            ref.append([G1.affine(p[name]) for name in snark._ORDER] + [G2.affine(p["PiB"])])
        k = len(wits)
        d_w = to_dev(np.concatenate(wl))
        for p in range(2):                                     # the satisfying witness and x_0 + 1
            out = d_words(108)
            check(L.b200_pinocchio_prove_witness_device(whole.pk.handle, sp.handle, d_w[4 * m * p:].data_ptr(), m,
                                                        out.data_ptr(), None))
            assert pin_affine(host(out)) == ref[p], f"witness_device {p}"
            g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
            check(L.b200_pinocchio_prove_witness(whole.pk.handle, sp.handle, ptr(wl[p]), m, ptr(g1), ptr(pb)))
            assert pin_affine(np.concatenate([g1, pb])) == ref[p], f"witness {p}"
        out = d_words(108 * k)
        check(L.b200_pinocchio_prove_witness_batch_device(whole.pk.handle, sp.handle, d_w.data_ptr(), m, k, out.data_ptr(),
                                                          None))
        assert pin_proofs(host(out), k) == ref, "batch"
        recs = d_words(256 * k * 3)
        for g, s in enumerate(shards):
            check(L.b200_pinocchio_prove_witness_batch_record_device(s.pk.handle, sp.handle, d_w.data_ptr(), m, k,
                                                                     recs[256 * k * g:].data_ptr(), None))
        out = d_words(108 * k)
        check(L.b200_pinocchio_finalize_records_batch_device(recs.data_ptr(), 3, k, out.data_ptr(), None))
        assert pin_proofs(host(out), k) == ref, "3-way records"
    finally:
        for key in keys:
            key.free()
        sp.free()


# ---- Groth16 -------------------------------------------------------------------------------------------------------
def g16_proofs(words, k):
    """k x 48 u64 (PiA | PiC | PiB) -> affine (PiA, PiB, PiC) per proof."""
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    out = []
    for p in range(k):
        q = words[48 * p:48 * p + 48]
        pa, pc = _unflatten_g1(q[:24])
        out.append((G1.affine(pa), G2.affine(_unflatten_g2(q[24:48])[0]), G1.affine(pc)))
    return out


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("n", SIZES)
def test_groth16_sharded_batch_px_division(L, n):
    """The world-8 records of b200_groth16_prove_witness_batch_partial_device (k = 1 and 3), finalised by
    b200_groth16_finalize_batch_device, equal b200_groth16_prove_witness_batch_device on the whole key, proof by proof;
    at n = 300 the batch also equals the known-discrete-log proof of each witness."""
    from gosnark_b200._lib import check, ptr
    inst = IrregularGroth16(n, n + 3, seed=n ^ 0xA5A5)
    m = inst.m
    pks = []
    try:
        pks.append(inst.load_pk())
        shards = [inst.load_pk(g, 8) for g in range(8)]
        pks += shards
        infos = []
        for h in shards:
            info = np.zeros(12, dtype=np.uint64)
            check(L.b200_groth16_shard_info(h, ptr(info)))
            infos.append(int(info[8]))
        assert sum(infos) >= 2, infos                          # so some rank's slice starts past h[0]
        wits = witnesses(inst.circuit, seed=n)
        rng = random.Random(n + 1)
        for k in (1, 3):
            ws = wits[:k] if k == 3 else [wits[1]]
            rs = [rng.randrange(R) for _ in range(k)]
            ss = [rng.randrange(R) for _ in range(k)]
            rl, sl = limbs(rs), limbs(ss)
            d_w = to_dev(np.concatenate([limbs(w) for w in ws]))
            out = d_words(48 * k)
            check(L.b200_groth16_prove_witness_batch_device(pks[0], inst.r1cs.handle, d_w.data_ptr(), m, k, ptr(rl),
                                                            ptr(sl), out.data_ptr(), None))
            ref = g16_proofs(host(out), k)
            parts = d_words(128 * k * 8)
            for g, h in enumerate(shards):
                check(L.b200_groth16_prove_witness_batch_partial_device(h, inst.r1cs.handle, d_w.data_ptr(), m, k, ptr(rl),
                                                                        ptr(sl), parts[128 * k * g:].data_ptr(), None))
            out = d_words(48 * k)
            check(L.b200_groth16_finalize_batch_device(shards[0], parts.data_ptr(), 8, k, out.data_ptr(), None))
            got = g16_proofs(host(out), k)
            for p in range(k):
                assert got[p] == ref[p], (k, p)
                if n < 1000:
                    a, b, c = inst.dlogs(ws[p], rs[p], ss[p])
                    assert ref[p] == (G1.affine(G1.mul_scalar(G1.G, a)), G2.affine(G2.mul_scalar(G2.G, b)),
                                      G1.affine(G1.mul_scalar(G1.G, c))), (k, p)
    finally:
        for h in pks:
            check(L.b200_pk_free(h))
        inst.r1cs.free()
