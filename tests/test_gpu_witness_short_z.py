"""GPU: witness-fed proving on circuits with m = n + 1 signals (len(Z) = n), whose quotient the device computes directly
and in batches: h = (x - n) q + kappa from the same front end as the m = n + 2 shape (csrc/qap_sparse.cuh).

The instances are synthetic.CircuitGroth16 / CircuitPinocchio with ``short_z=True``: a real trusted setup of the m = n + 1
chain, known discrete logs, and a real Vk.  Every witness-fed proof is held against the px-fed entry on the px of
b200_qap_px (affine: the two entries' MSMs may leave different Jacobian representatives), against the known-discrete-log proof where the witness satisfies the circuit,
and against the real Vk.  The Go binary's own m = n + 1 circuits (x3x5, chain21) are covered by the golden tests of the
witness-fed entries, which take this branch."""
import ctypes
import random
import threading

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
G1, G2 = o.BN.G1, o.BN.G2
R = o.R
PIN_ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


_g16, _pin = {}, {}


def g16(n):
    from gosnark_b200.synthetic import CircuitGroth16
    if n not in _g16:
        _g16[n] = CircuitGroth16(n=n, short_z=True)
        assert _g16[n].m == n + 1 and _g16[n].z.shape[0] == n
    return _g16[n]


def pin(n):
    from gosnark_b200.synthetic import CircuitPinocchio
    if n not in _pin:
        _pin[n] = CircuitPinocchio(n, short_z=True)
        assert _pin[n].m == n + 1 and _pin[n].pk["G1T"].shape[0] == n
    return _pin[n]


def _p(a):
    from gosnark_b200._lib import ptr
    return ptr(a)


def limbs(vals):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs(list(vals))


def to_dev(arr):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def with_config(L, fn, ctx=0, acc=0, t=0):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    try:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, ctx))
        check(L.b200_config(_lib.CFG_ACC_MODE, acc))
        check(L.b200_config(_lib.CFG_TABLE_WINDOWS, t))
        return fn()
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))
        check(L.b200_config(_lib.CFG_ACC_MODE, 0))
        check(L.b200_config(_lib.CFG_TABLE_WINDOWS, 0))


def witnesses(syn, k, seed=0):
    """k witnesses of syn's circuit (ints) and whether each satisfies it: p = 1 has one signal off, p = 4 is random, the
    others are distinct satisfying ones."""
    from gosnark_b200.synthetic import SyntheticCircuit
    out, sat = [], []
    for p in range(k):
        w = list(SyntheticCircuit(syn.n, seed=0x5407 + 977 * seed + p, short_z=True).witness)
        if p == 1:
            w[syn.n // 2 + 1] = (w[syn.n // 2 + 1] + 1) % R
        elif p == 4:
            rng = random.Random(seed)
            w = [1] + [rng.randrange(R) for _ in range(syn.m - 1)]
        out.append(w)
        sat.append(p not in (1, 4))
    return out, sat


def blindings(k, seed=0):
    return ([((0x1234567 * (p + 3) + seed) << 180 | p) % R for p in range(k)],
            [((0x7654321 * (p + 5) + seed) << 170 | p) % R for p in range(k)])


# ---- Groth16 ----------------------------------------------------------------------------------------------------------
def g_split(words):
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    pa, pc = _unflatten_g1(words[:24])
    return pa, _unflatten_g2(words[24:48])[0], pc


def g_affine(p):
    pa, pb, pc = p
    return G1.affine(pa), G2.affine(pb), G1.affine(pc)


def g_expected(dlogs):
    a, b, c = dlogs
    return G1.affine(G1.mul_scalar(G1.G, a)), G2.affine(G2.mul_scalar(G2.G, b)), G1.affine(G1.mul_scalar(G1.G, c))


def g_verify(syn, proof, public):
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    ok = ctypes.c_int(0)
    pa, pb, pc = proof
    check(syn_lib().b200_groth16_verify(ptr(syn.ic), syn.npublic + 1, ptr(syn.alpha1), ptr(syn.beta2), ptr(syn.gamma2),
                                        ptr(syn.delta2), ptr(_flatten_g1([pa])), ptr(_flatten_g2([pb])), ptr(_flatten_g1([pc])),
                                        ptr(ints_to_limbs(public)), len(public), ctypes.byref(ok)))
    return bool(ok.value)


def syn_lib():
    from gosnark_b200._lib import lib
    return lib()


def g_px_device(L, pk, w, px, r, s):
    import torch
    from gosnark_b200._lib import check
    d_w, d_px = to_dev(w), to_dev(px)
    d_out = torch.full((48,), -1, dtype=torch.int64, device="cuda")
    check(L.b200_groth16_prove_device(pk, d_w.data_ptr(), w.shape[0], d_px.data_ptr(), px.shape[0], _p(limbs([r])),
                                      _p(limbs([s])), d_out.data_ptr(), None))
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint64).copy()


def g_witness_device(L, pk, r1cs, w, r, s, stream=None):
    import torch
    from gosnark_b200._lib import check
    d_w = to_dev(w)
    d_out = torch.full((48,), -1, dtype=torch.int64, device="cuda")
    check(L.b200_groth16_prove_witness_device(pk, r1cs, d_w.data_ptr(), w.shape[0], _p(limbs([r])), _p(limbs([s])),
                                              d_out.data_ptr(), None if stream is None else stream.cuda_stream))
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint64).copy()


def g_witness_host(L, pk, r1cs, w, r, s):
    from gosnark_b200._lib import check
    pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
    check(L.b200_groth16_prove_witness(pk, r1cs, _p(w), w.shape[0], _p(limbs([r])), _p(limbs([s])), _p(pa), _p(pb), _p(pc)))
    return g_split(np.concatenate([pa, pc, pb]))


def g_batch_device(L, pk, r1cs, d_w, m, rs, ss, d_out):
    return L.b200_groth16_prove_witness_batch_device(pk, r1cs, d_w.data_ptr(), m, len(rs), _p(limbs(rs)), _p(limbs(ss)),
                                                     d_out.data_ptr(), None)


def g_batch(L, pk, r1cs, wits, m, rs, ss):
    import torch
    from gosnark_b200._lib import check
    k = len(rs)
    d_out = torch.full((48 * k,), -1, dtype=torch.int64, device="cuda")
    check(g_batch_device(L, pk, r1cs, to_dev(limbs([v for w in wits for v in w])), m, rs, ss, d_out))
    torch.cuda.synchronize()
    raw = d_out.cpu().numpy().view(np.uint64)
    return [g_split(raw[48 * p:48 * p + 48]) for p in range(k)]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("n,acc,t", [((1 << 12) + 1, 1, 0), ((1 << 12) + 1, 2, 0), ((1 << 12) + 1, 0, 1), (1 << 16, 0, 0),
                                     (1 << 20, 0, 0)],
                         ids=["4097-affine", "4097-xyzz", "4097-one-table-window", "65536", "1048576"])
def test_groth16_single_proofs(L, n, acc, t):
    """The device witness entry equals (affine) b200_qap_px followed by the px-fed entry, is the known-discrete-log
    proof and verifies; the host entry agrees.  An unsatisfied witness (one signal off; at 2^12 + 1
    also a random one) gets the px-fed proof of its own px and is refused."""
    from gosnark_b200._lib import check
    syn = g16(n)
    pk = with_config(L, syn.load_pk, acc=acc, t=t)
    try:
        h = syn.r1cs.handle
        dev = g_witness_device(L, pk, h, syn.w, syn.r, syn.s)
        assert g_affine(g_split(dev)) == g_affine(g_split(g_px_device(L, pk, syn.w, syn.px, syn.r, syn.s)))
        assert g_affine(g_split(dev)) == g_expected(syn.expected_dlogs())
        assert g_verify(syn, g_split(dev), syn.circuit.public_signals)
        assert g_affine(g_witness_host(L, pk, h, syn.w, syn.r, syn.s)) == g_affine(g_split(dev))
        bad = [list(syn.circuit.witness)]
        bad[0][n // 2 + 1] = (bad[0][n // 2 + 1] + 1) % R
        if n < (1 << 16):
            rng = random.Random(n)
            bad.append([1] + [rng.randrange(R) for _ in range(syn.m - 1)])
        for wi in bad:
            w = limbs(wi)
            dev = g_witness_device(L, pk, h, w, syn.r, syn.s)
            assert g_affine(g_split(dev)) == g_affine(g_split(g_px_device(L, pk, w, syn.px_of(w), syn.r, syn.s)))
            assert not g_verify(syn, g_split(dev), [wi[1]])
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("n", [(1 << 12) + 1, 1 << 16])
def test_groth16_batches(L, n):
    """k in {1, 2, 5, 8}, satisfied and unsatisfied witnesses mixed: proof p equals the single entry's (affine), the
    known-discrete-log proof when w_p satisfies the circuit, and verifies exactly then."""
    from gosnark_b200._lib import check
    syn = g16(n)
    pk = syn.load_pk()
    try:
        for k in (1, 2, 5, 8):
            wits, sat = witnesses(syn, k, seed=k)
            rs, ss = blindings(k, seed=k)
            got = g_batch(L, pk, syn.r1cs.handle, wits, syn.m, rs, ss)
            for p in range(k):
                single = g_split(g_witness_device(L, pk, syn.r1cs.handle, limbs(wits[p]), rs[p], ss[p]))
                assert g_affine(got[p]) == g_affine(single), (k, p)
                if sat[p]:
                    assert g_affine(got[p]) == g_expected(syn.expected_dlogs(wits[p], rs[p], ss[p])), (k, p)
                if p < 3:
                    assert g_verify(syn, got[p], [wits[p][1]]) == sat[p], (k, p)
    finally:
        check(L.b200_pk_free(pk))


def _launches(L, fn):
    from gosnark_b200._lib import check
    out = (ctypes.c_double * 8)()
    check(L.b200_profile_read(out))
    fn()
    check(L.b200_profile_read(out))
    return int(out[6])


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
    64 Ki (multi-block scan); no tail chunking below 65536 rows."""
    return int(k * (1 << (c - 1)) + 1 > 65536) - int((1 << (c - 1)) + 1 > 65536)


# The launches the m = n + 1 branch adds to a call of the m = n + 2 one: k_short_z_dot (the shifted store takes the place
# of k_quotient_store in a batch, of k_poly_store in a single proof).
SHORT_Z_EXTRA_LAUNCHES = 1


@pytest.mark.timeout(1200)
def test_groth16_batch_launches(L):
    """From b200_profile_read at n = 2^12: a batch of 8 issues the launches of a batch of one plus the batched MSM's
    extras, and at most the launches of an m = n + 2 batch of 8 at the same n plus SHORT_Z_EXTRA_LAUNCHES; a single proof
    at most the m = n + 2 single proof's plus the same."""
    import torch
    from gosnark_b200._lib import check
    from gosnark_b200.synthetic import CircuitGroth16
    n = 1 << 12
    short, full = g16(n), CircuitGroth16(n=n)
    pks = [short.load_pk(), full.load_pk()]
    try:
        counts = []
        for syn, pk in zip((short, full), pks):
            wits = [list(syn.circuit.witness)] * 8
            d_w = to_dev(limbs([v for w in wits for v in w]))
            d_out = torch.zeros(48 * 8, dtype=torch.int64, device="cuda")

            def batch(k):
                rs, ss = blindings(k)
                check(g_batch_device(L, pk, syn.r1cs.handle, d_w, syn.m, rs, ss, d_out))

            def single():
                check(L.b200_groth16_prove_witness_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, _p(limbs([syn.r])),
                                                          _p(limbs([syn.s])), d_out.data_ptr(), None))
            for k in (1, 8):            # warm-up: scratch and domains
                batch(k)
            single()
            torch.cuda.synchronize()
            counts.append((_launches(L, lambda: batch(1)), _launches(L, lambda: batch(8)), _launches(L, single)))
            torch.cuda.synchronize()
        (s1, s8, ss1), (f1, f8, fs1) = counts
        c_ab, c_ch = pick_window_bits(short.m + 3), pick_window_bits(2 * short.m - 2)
        assert s8 == s1 + msm_extras(8, c_ab) + msm_extras(8, c_ch), counts
        assert s8 <= f8 + SHORT_Z_EXTRA_LAUNCHES, counts
        assert ss1 <= fs1 + SHORT_Z_EXTRA_LAUNCHES, counts
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("world", [2, 3])
def test_groth16_shards(L, world):
    """Key shards emulated on one GPU: every rank's partial records -> b200_groth16_finalize_batch_device equal the
    unsharded batch, and the single device entry's records the same way."""
    import torch
    from gosnark_b200._lib import check
    n = 1 << 10
    syn = g16(n)
    pk1 = syn.load_pk()
    pks = [syn.load_pk(g, world) for g in range(world)]
    try:
        for k in (1, 3, 5):
            wits, sat = witnesses(syn, k, seed=world * 10 + k)
            rs, ss = blindings(k, seed=k)
            d_w = to_dev(limbs([v for w in wits for v in w]))
            ref = g_batch(L, pk1, syn.r1cs.handle, wits, syn.m, rs, ss)
            parts = torch.full((128 * world * k,), -1, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            for g, pk in enumerate(pks):
                check(L.b200_groth16_prove_witness_batch_partial_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, k,
                                                                        _p(limbs(rs)), _p(limbs(ss)),
                                                                        parts[128 * k * g:].data_ptr(), None))
            d_out = torch.full((48 * k,), -1, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            check(L.b200_groth16_finalize_batch_device(pks[0], parts.data_ptr(), world, k, d_out.data_ptr(), None))
            torch.cuda.synchronize()
            raw = d_out.cpu().numpy().view(np.uint64)
            for p in range(k):
                assert g_affine(g_split(raw[48 * p:48 * p + 48])) == g_affine(ref[p]), (k, p)
                if sat[p]:
                    assert g_affine(ref[p]) == g_expected(syn.expected_dlogs(wits[p], rs[p], ss[p])), (k, p)
    finally:
        for pk in pks + [pk1]:
            check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_groth16_two_contexts_in_flight(L):
    """Keys of contexts 0 and 1 on ONE m = n + 1 R1CS handle, device witness entries on two torch streams interleaved, a
    satisfied and an unsatisfied witness: each proof equals its own px-fed expectation."""
    import torch
    from gosnark_b200._lib import check
    n = (1 << 12) + 1
    syn = g16(n)
    pks = [with_config(L, syn.load_pk, ctx=c) for c in range(2)]
    try:
        wits, _ = witnesses(syn, 2, seed=77)
        ws = [limbs(w) for w in wits]
        want = [g_px_device(L, pks[c], ws[c], syn.px_of(ws[c]), syn.r, syn.s) for c in range(2)]
        d_ws = [to_dev(w) for w in ws]
        outs = [torch.full((48,), -1, dtype=torch.int64, device="cuda") for _ in range(2)]
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        for _ in range(3):
            for c in range(2):
                check(L.b200_groth16_prove_witness_device(pks[c], syn.r1cs.handle, d_ws[c].data_ptr(), syn.m,
                                                          _p(limbs([syn.r])), _p(limbs([syn.s])), outs[c].data_ptr(),
                                                          streams[c].cuda_stream))
        torch.cuda.synchronize()
        for c in range(2):
            assert g_affine(g_split(outs[c].cpu().numpy().view(np.uint64))) == g_affine(g_split(want[c])), c
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


# ---- Pinocchio --------------------------------------------------------------------------------------------------------
def p_split(words):
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    proof = dict(zip(PIN_ORDER, _unflatten_g1(words[:84])))
    proof["PiB"] = _unflatten_g2(words[84:108])[0]
    return proof


def p_affine(proof):
    return tuple(G1.affine(proof[k]) for k in PIN_ORDER) + (G2.affine(proof["PiB"]),)


def p_expected(dlogs):
    return tuple(G1.affine(G1.mul_scalar(G1.G, dlogs[k])) for k in PIN_ORDER) + (G2.affine(G2.mul_scalar(G2.G, dlogs["PiB"])),)


def p_px_device(L, pk, w, px):
    import torch
    from gosnark_b200._lib import check
    d_w, d_px = to_dev(w), to_dev(px)
    d_out = torch.full((108,), -1, dtype=torch.int64, device="cuda")
    check(L.b200_pinocchio_prove_device(pk, d_w.data_ptr(), w.shape[0], d_px.data_ptr(), px.shape[0], d_out.data_ptr(), None))
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint64).copy()


def p_witness_device(L, pk, r1cs, w, stream=None):
    import torch
    from gosnark_b200._lib import check
    d_w = to_dev(w)
    d_out = torch.full((108,), -1, dtype=torch.int64, device="cuda")
    check(L.b200_pinocchio_prove_witness_device(pk, r1cs, d_w.data_ptr(), w.shape[0], d_out.data_ptr(),
                                                None if stream is None else stream.cuda_stream))
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint64).copy()


def p_batch(L, pk, r1cs, wits, m):
    import torch
    from gosnark_b200._lib import check
    k = len(wits)
    d_out = torch.full((108 * k,), -1, dtype=torch.int64, device="cuda")
    check(L.b200_pinocchio_prove_witness_batch_device(pk, r1cs, to_dev(limbs([v for w in wits for v in w])).data_ptr(), m, k,
                                                      d_out.data_ptr(), None))
    torch.cuda.synchronize()
    raw = d_out.cpu().numpy().view(np.uint64)
    return [p_split(raw[108 * p:108 * p + 108]) for p in range(k)]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("n,acc", [((1 << 12) + 1, 1), ((1 << 12) + 1, 2), (1 << 16, 0)], ids=["4097-affine", "4097-xyzz", "65536"])
def test_pinocchio_single_proofs(L, n, acc):
    """Equal (affine) to the px-fed entry on b200_qap_px's px, the known-discrete-log proof, accepted by the real Vk; an
    unsatisfied witness gets its own px-fed proof and is refused."""
    from gosnark_b200._lib import check
    syn = pin(n)
    pk = with_config(L, syn.load_pk, acc=acc)
    try:
        h = syn.r1cs.handle
        dev = p_witness_device(L, pk, h, syn.w)
        assert p_affine(p_split(dev)) == p_affine(p_split(p_px_device(L, pk, syn.w, syn.px)))
        assert p_affine(p_split(dev)) == p_expected(syn.expected_dlogs())
        assert syn.verify(p_split(dev))
        wi = list(syn.circuit.witness)
        wi[n // 2 + 1] = (wi[n // 2 + 1] + 1) % R
        w = limbs(wi)
        dev = p_witness_device(L, pk, h, w)
        assert p_affine(p_split(dev)) == p_affine(p_split(p_px_device(L, pk, w, syn.px_of(w))))
        assert not syn.verify(p_split(dev), [wi[1]])
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(1800)
def test_pinocchio_batches_and_launches(L):
    """k in {1, 2, 5, 8} at n = 2^12 + 1: proof p equals the single entry's and, for a satisfying witness, the
    known-discrete-log proof; a batch of 8 issues the launches of a batch of one plus the batched MSM's extras."""
    import torch
    from gosnark_b200._lib import check
    n = (1 << 12) + 1
    syn = pin(n)
    pk = syn.load_pk()
    try:
        for k in (1, 2, 5, 8):
            wits, sat = witnesses(syn, k, seed=k)
            got = p_batch(L, pk, syn.r1cs.handle, wits, syn.m)
            for p in range(k):
                assert p_affine(got[p]) == p_affine(p_split(p_witness_device(L, pk, syn.r1cs.handle, limbs(wits[p])))), (k, p)
                if sat[p]:
                    assert p_affine(got[p]) == p_expected(syn.expected_dlogs(wits[p])), (k, p)
        wits, _ = witnesses(syn, 8, seed=3)
        d_w = to_dev(limbs([v for w in wits for v in w]))
        d_out = torch.zeros(108 * 8, dtype=torch.int64, device="cuda")

        def batch(k):
            check(L.b200_pinocchio_prove_witness_batch_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, k, d_out.data_ptr(), None))
        for k in (1, 8):          # warm-up: scratch and domains
            batch(k)
        c1, c8 = _launches(L, lambda: batch(1)), _launches(L, lambda: batch(8))
        extras = msm_extras(8, pick_window_bits(syn.m)) + msm_extras(8, pick_window_bits(syn.m - 2)) + \
            msm_extras(8, pick_window_bits(n))
        assert c8 == c1 + extras, (c1, c8)
        torch.cuda.synchronize()
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("world", [2, 3])
def test_pinocchio_shards(L, world):
    """Every rank's k records -> b200_pinocchio_finalize_records_batch_device equal the unsharded batch."""
    import torch
    from gosnark_b200._lib import check
    n = 1 << 10
    syn = pin(n)
    pk1 = syn.load_pk()
    pks = [syn.load_pk(g, world) for g in range(world)]
    try:
        for k in (1, 3, 5):
            wits, _ = witnesses(syn, k, seed=world * 10 + k)
            d_w = to_dev(limbs([v for w in wits for v in w]))
            ref = p_batch(L, pk1, syn.r1cs.handle, wits, syn.m)
            recs = torch.full((256 * world * k,), -1, dtype=torch.int64, device="cuda")
            d_out = torch.full((108 * k,), -1, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            for g, pk in enumerate(pks):
                check(L.b200_pinocchio_prove_witness_batch_record_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, k,
                                                                         recs[256 * k * g:].data_ptr(), None))
            check(L.b200_pinocchio_finalize_records_batch_device(recs.data_ptr(), world, k, d_out.data_ptr(), None))
            torch.cuda.synchronize()
            raw = d_out.cpu().numpy().view(np.uint64)
            for p in range(k):
                assert p_affine(p_split(raw[108 * p:108 * p + 108])) == p_affine(ref[p]), (k, p)
    finally:
        for pk in pks + [pk1]:
            check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_pinocchio_two_contexts_in_flight(L):
    """Keys of contexts 0 and 1 on one m = n + 1 R1CS handle, proofs in flight on two host threads: each equals its
    px-fed expectation."""
    from gosnark_b200._lib import check
    n = (1 << 12) + 1
    syn = pin(n)
    pks = [with_config(L, syn.load_pk, ctx=c) for c in range(2)]
    try:
        wits, _ = witnesses(syn, 2, seed=91)
        ws = [limbs(w) for w in wits]
        want = [p_px_device(L, pks[c], ws[c], syn.px_of(ws[c])) for c in range(2)]
        got, errs = [None, None], []

        def run(c):
            try:
                from gosnark_b200._lib import ptr
                g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
                for _ in range(3):
                    check(L.b200_pinocchio_prove_witness(pks[c], syn.r1cs.handle, ptr(ws[c]), syn.m, ptr(g1), ptr(pb)))
                got[c] = p_split(np.concatenate([g1, pb]))
            except Exception as e:      # noqa: BLE001 - reported below
                errs.append(e)
        th = [threading.Thread(target=run, args=(c,)) for c in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errs, errs
        for c in range(2):
            assert p_affine(got[c]) == p_affine(p_split(want[c])), c
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))
