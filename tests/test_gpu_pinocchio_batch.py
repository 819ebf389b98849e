"""GPU: batched witness-fed Pinocchio proving (include/b200snark.h: b200_pinocchio_prove_witness_batch,
b200_pinocchio_prove_witness_batch_device): k proofs under one key in one set of launches.  Proof p of a batch is
compared, on affine coordinates, with what b200_pinocchio_prove_witness_device gives for w_p and, for satisfying
witnesses, with the known-discrete-log proof of synthetic.CircuitPinocchio."""
import threading

import numpy as np
import pytest

from test_gpu_pinocchio_witness import (EINVAL, ERANGE, ORDER, R, _golden, _launches, _p, affine, circuit, expected, limbs,
                                        load_pk, pinocchio_pk, pk_bytes, split, to_dev, unsatisfied, witness_device)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


def witnesses(syn, k, seed=0):
    """k witnesses of syn's circuit (ints) and whether each satisfies it: every fifth has one signal off, every seventh
    is random, the others are distinct satisfying ones."""
    from gosnark_b200.synthetic import SyntheticCircuit
    out, sat = [], []
    for p in range(k):
        if p % 5 == 3:
            out.append(unsatisfied(syn, "one"))
        elif p % 7 == 5:
            out.append(unsatisfied(syn, "every"))
        else:
            out.append(SyntheticCircuit(syn.n, seed=0xBA7C0 + 977 * seed + p).witness)
        sat.append(p % 5 != 3 and p % 7 != 5)
    return out, sat


def flat(wits):
    return limbs([v for w in wits for v in w])


def batch_device(L, pk, r1cs, d_w, m, k, d_out, stream=None):
    return L.b200_pinocchio_prove_witness_batch_device(pk, r1cs, d_w.data_ptr(), m, k, d_out.data_ptr(),
                                                       None if stream is None else stream.cuda_stream)


def run_device_batch(L, pk, r1cs, wl, m, k, stream=None):
    import torch
    from gosnark_b200._lib import check
    d_out = torch.full((108 * k,), -1, dtype=torch.int64, device="cuda")
    check(batch_device(L, pk, r1cs, to_dev(wl), m, k, d_out, stream))
    torch.cuda.synchronize()
    raw = d_out.cpu().numpy().view(np.uint64)
    return [split(raw[108 * p:108 * p + 108]) for p in range(k)]


def batch_host(L, pk, r1cs, wl, m, k):
    from gosnark_b200._lib import check
    g1, pb = np.zeros(84 * k, np.uint64), np.zeros(24 * k, np.uint64)
    check(L.b200_pinocchio_prove_witness_batch(pk, r1cs, _p(wl), m, k, _p(g1), _p(pb)))
    return [split(np.concatenate([g1[84 * p:84 * p + 84], pb[24 * p:24 * p + 24]])) for p in range(k)]


def check_batch(L, syn, pk, proofs, wits, sat, singles=None):
    """Proof p is the single entry's proof of w_p (all p, or those listed) and, for a satisfying witness, the
    known-discrete-log proof."""
    for p, got in enumerate(proofs):
        if sat[p]:
            assert affine(got) == expected(syn.expected_dlogs(wits[p])), p
        if singles is None or p in singles or not sat[p]:
            assert affine(got) == affine(witness_device(L, pk, syn.r1cs.handle, limbs(wits[p]))), p


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("n,acc,ks", [(1 << 10, 0, (1, 2, 3, 8, 33)), ((1 << 12) + 2, 1, (1, 2, 3, 8, 33)),
                                      ((1 << 12) + 2, 2, (2, 3)), (1 << 16, 0, (4,))],
                         ids=["1024", "4098-affine", "4098-xyzz", "65536"])
def test_sizes_and_entries(L, n, acc, ks):
    """Satisfied and unsatisfied witnesses mixed; the host entry and the device entry (library stream and a torch side
    stream) agree; the first proof of a batch that holds a satisfying witness verifies under the real Vk."""
    import torch
    from gosnark_b200._lib import check
    syn = circuit(n)
    pk = load_pk(L, syn, acc=acc)
    try:
        for k in ks:
            wits, sat = witnesses(syn, k, seed=k)
            wl = flat(wits)
            dev = run_device_batch(L, pk, syn.r1cs.handle, wl, syn.m, k)
            check_batch(L, syn, pk, dev, wits, sat, singles=None if k <= 8 else {0, k // 2, k - 1})
            for name, other in (("host", batch_host(L, pk, syn.r1cs.handle, wl, syn.m, k)),
                                ("side-stream", run_device_batch(L, pk, syn.r1cs.handle, wl, syn.m, k, torch.cuda.Stream()))):
                assert [affine(p) for p in other] == [affine(p) for p in dev], (name, k)
            assert syn.verify(dev[0], [wits[0][1]])
            if k > 3:
                assert not syn.verify(dev[3], [wits[3][1]])
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.parametrize("name", ["x3x5", "chain21"])
def test_go_binary_circuit_batch_equals_its_singles(L, golden_dir, name):
    """len(Z) = n: px and the division once per witness.  The golden witness and two others in one batch."""
    from gosnark_b200 import snark
    from gosnark_b200._lib import ints_to_limbs
    from gosnark_b200.bn128 import reduce_scalar
    from gosnark_b200.r1csqap import SparseR1CS
    from oracle import ref_py as o
    g = _golden(golden_dir, name)
    cc = g["compiledcircuit"]
    a, b, c = cc["R1CS"]["A"], cc["R1CS"]["B"], cc["R1CS"]["C"]
    n, m = len(a), len(a[0])
    sp = SparseR1CS(n, m, (a, b, c))
    dpk = snark.DeviceProvingKey(pinocchio_pk(g["pinocchio_setup"]), m, cc["NPublic"])
    try:
        w = [reduce_scalar(x) for x in g["witness"]]
        off = list(w)
        off[-1] = (off[-1] + 1) % R
        ws = np.stack([ints_to_limbs(v) for v in (w, off, w)])
        got = dpk.prove_witness_batch_limbs(sp, ws)
        for p in range(3):
            assert affine(got[p]) == affine(dpk.prove_witness_limbs(sp, ws[p])), p
        ref = g["pinocchio_proofs"]
        for kk in ORDER:
            assert o.BN.G1.affine(got[0][kk]) == o.BN.G1.affine(tuple(ref[kk])), kk
        assert affine(got[0]) == affine(got[2]) != affine(got[1])
    finally:
        dpk.free()
        sp.free()


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


@pytest.mark.timeout(900)
def test_launch_count_does_not_grow_with_k(L):
    """From b200_profile_read: a batch of k issues the launches of a batch of one plus the batched MSM's extras of its
    three sorts (w over m terms, w[l+1..) over m - l - 1, the quotients over len(G1T)), and fewer than k single proofs."""
    import torch
    from gosnark_b200._lib import check
    n = (1 << 12) + 2
    syn = circuit(n)
    pk = load_pk(L, syn)
    try:
        wits, _ = witnesses(syn, 8, seed=3)
        d_w = to_dev(flat(wits))
        d_out = torch.zeros(108 * 8, dtype=torch.int64, device="cuda")
        l1 = syn.npublic + 1
        cs = [pick_window_bits(t) for t in (syn.m, syn.m - l1, syn.pk["G1T"].shape[0])]

        def batch(k):
            check(batch_device(L, pk, syn.r1cs.handle, d_w, syn.m, k, d_out))
        for k in (1, 8):          # warm-up: scratch and domains
            batch(k)
        base = _launches(L, lambda: batch(1))
        single = _launches(L, lambda: check(L.b200_pinocchio_prove_witness_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m,
                                                                                 d_out.data_ptr(), None)))
        for k in (2, 8):
            got = _launches(L, lambda: batch(k))
            assert got == base + sum(msm_extras(k, c) for c in cs), (k, got, base)
            assert got < k * single, (k, got, single)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_scratch_regrowth_and_two_contexts(L):
    """k = 2, 8, 3 on one stream with no host synchronisation between the calls: b200_pk_device_bytes grows at the first
    call and at k = 8, then stays, and every proof is right.  Then batches on a context-0 and a context-1 key in flight
    together on one R1CS handle, and the host entry from two threads."""
    import torch
    from gosnark_b200._lib import check
    n = 1 << 10
    syn = circuit(n)
    pks = [load_pk(L, syn, ctx=c) for c in range(2)]
    try:
        wits, sat = witnesses(syn, 8, seed=5)
        want = [affine(witness_device(L, pks[0], syn.r1cs.handle, limbs(w))) for w in wits]
        d_w = to_dev(flat(wits))
        st = torch.cuda.Stream()
        sizes, outs = [pk_bytes(L, pks[0])], []
        for k in (2, 8, 3):
            d = torch.zeros(108 * k, dtype=torch.int64, device="cuda")
            check(batch_device(L, pks[0], syn.r1cs.handle, d_w, syn.m, k, d, st))
            outs.append((k, d))
            sizes.append(pk_bytes(L, pks[0]))
        assert sizes[0] < sizes[1] < sizes[2] == sizes[3], sizes
        torch.cuda.synchronize()
        for k, d in outs:
            raw = d.cpu().numpy().view(np.uint64)
            assert [affine(split(raw[108 * p:108 * p + 108])) for p in range(k)] == want[:k], k
        # two contexts in flight
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        k = 3
        d_c = [to_dev(flat(wits[c * k:(c + 1) * k])) for c in range(2)]
        for c in range(2):      # the first call per (R1CS, context) builds its workspace and may synchronise
            check(batch_device(L, pks[c], syn.r1cs.handle, d_c[c], syn.m, k, torch.zeros(108 * k, dtype=torch.int64, device="cuda"), streams[c]))
        torch.cuda.synchronize()
        outs = {}
        for j in range(3):
            for c in range(2):
                outs[(j, c)] = torch.zeros(108 * k, dtype=torch.int64, device="cuda")
                check(batch_device(L, pks[c], syn.r1cs.handle, d_c[c], syn.m, k, outs[(j, c)], streams[c]))
        torch.cuda.synchronize()
        for (j, c), d in outs.items():
            raw = d.cpu().numpy().view(np.uint64)
            assert [affine(split(raw[108 * p:108 * p + 108])) for p in range(k)] == want[c * k:(c + 1) * k], (j, c)
        results, errs = {}, []

        def worker(c):
            try:
                for j in range(3):
                    results[(c, j)] = batch_host(L, pks[c], syn.r1cs.handle, flat(wits[c * k:(c + 1) * k]), syn.m, k)
            except Exception as e:   # noqa: BLE001 - reported below
                errs.append(e)
        ths = [threading.Thread(target=worker, args=(c,)) for c in range(2)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        assert not errs, errs
        for (c, j), proofs in results.items():
            assert [affine(p) for p in proofs] == want[c * k:(c + 1) * k], (c, j)
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


def load_raw(L, syn, m, npublic, g1t, z):
    """A Pinocchio key over the first m points of syn's sets, with the given NPublic, G1T prefix and Z (limbs)."""
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    p = syn.pk
    h = _lib._h(0)
    check(L.b200_pinocchio_pk_load(_p(p["A"]), _p(p["Ap"]), _p(p["B"]), _p(p["Bp"]), _p(p["C"]), _p(p["Cp"]), _p(p["Kp"]), m,
                                   _p(p["G1T"]), g1t, _p(z), z.shape[0], npublic, 0, h))
    return h.value


@pytest.mark.timeout(600)
def test_every_signal_public(L):
    """NPublic + 1 == NVars: the key holds no A and no Ap set (snark.go:265-268 sum over nothing), so PiA and PiAp are the
    point at infinity, all-zero words, in every proof of a batch as in the single entry - also in a scratch that an
    earlier, larger batch has written."""
    from gosnark_b200._lib import check
    syn = circuit(1 << 6)
    pk = load_raw(L, syn, syn.m, syn.m - 1, syn.pk["G1T"].shape[0], syn.z)
    try:
        wits, _ = witnesses(syn, 3, seed=21)
        singles = [witness_device(L, pk, syn.r1cs.handle, limbs(w)) for w in wits]
        assert singles[0]["PiA"] == (0, 0, 0) and singles[0]["PiAp"] == (0, 0, 0)
        zero = (0, 0), (0, 0), (0, 0)
        assert singles[0]["PiC"] != (0, 0, 0) and singles[0]["PiB"] != zero
        for k in (3, 1, 3):
            for got in (run_device_batch(L, pk, syn.r1cs.handle, flat(wits[:k]), syn.m, k),
                        batch_host(L, pk, syn.r1cs.handle, flat(wits[:k]), syn.m, k)):
                for p in range(k):
                    assert got[p]["PiA"] == (0, 0, 0) and got[p]["PiAp"] == (0, 0, 0), (k, p)
                    assert affine(got[p]) == affine(singles[p]), (k, p)
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(600)
def test_transform_bound_is_refused_on_its_own(L):
    """3k * 2N >= 2^32 transform elements with every sort far below 2^31 entries: a circuit of 2^16 constraints over 8
    signals whose key has len(Z) = 2n - 1, so one quotient coefficient and one G1T point.  (With m ~ n, as in every other
    circuit here, the sort-entry bound is reached first.)  Refused before anything is allocated."""
    import torch
    from gosnark_b200._lib import check, lib
    from gosnark_b200.r1csqap import SparseR1CS
    syn = circuit(1 << 6)
    n, m = 1 << 16, 8
    rowptr = np.arange(n + 1, dtype=np.uint32)
    col = (np.arange(n, dtype=np.uint32) % m).astype(np.uint32)
    ones = np.zeros((n, 4), dtype=np.uint64)
    ones[:, 0] = 1
    sp = SparseR1CS(n, m, [(rowptr, col, ones)] * 3)
    z = np.zeros((2 * n - 1, 4), dtype=np.uint64)
    z[:, 0] = 1
    pk = load_raw(L, syn, m, 1, 1, z)
    try:
        k = (1 << 32) // (6 * n) + 1                         # the first k with 6 k N >= 2^32
        assert 6 * k * n >= 1 << 32 > 6 * (k - 1) * n and k * 32 * m < 1 << 31
        d = torch.zeros(8, dtype=torch.int64, device="cuda")   # never read: the call is refused first
        before = pk_bytes(L, pk)
        assert L.b200_pinocchio_prove_witness_batch_device(pk, sp.handle, d.data_ptr(), m, k, d.data_ptr(), None) == EINVAL
        assert b"transform elements" in lib().b200_last_error()
        g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
        assert L.b200_pinocchio_prove_witness_batch(pk, sp.handle, _p(g1), m, k, _p(g1), _p(pb)) == EINVAL
        assert b"transform elements" in lib().b200_last_error()
        assert pk_bytes(L, pk) == before
    finally:
        check(L.b200_pk_free(pk))
        sp.free()


@pytest.mark.timeout(600)
def test_errors(L):
    """Each B200_EINVAL leaves b200_pk_device_bytes unchanged; a witness entry >= r in witness 2 of 5 gives B200_ERANGE on
    the host entry, leaves the outputs untouched, and the next batch on the key is right; a Groth16 key is refused."""
    import torch
    from gosnark_b200._lib import check
    from gosnark_b200.synthetic import CircuitGroth16
    syn, small = circuit(1 << 10), circuit(1 << 6)
    groth = CircuitGroth16(n=1 << 6)
    pk, pk_g = load_pk(L, syn), groth.load_pk()
    pk_shard = load_pk(L, syn, rank=0, world=2)
    try:
        m, h, k = syn.m, syn.r1cs.handle, 5
        wits, sat = witnesses(syn, k, seed=9)
        wl = flat(wits)
        d_w = to_dev(wl)
        d_out = torch.zeros(108 * k, dtype=torch.int64, device="cuda")
        g1, pb = np.zeros(84 * k, np.uint64), np.zeros(24 * k, np.uint64)
        W, O = d_w.data_ptr(), d_out.data_ptr()
        before = pk_bytes(L, pk)
        too_many = (1 << 31) // (syn.m * 8)                  # k * nwin * m sort entries reach 2^31 well before this
        bad = [
            L.b200_pinocchio_prove_witness_batch(pk, h, _p(wl), m, 0, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness_batch(pk + 1000, h, _p(wl), m, k, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness_batch(pk, h + 1000, _p(wl), m, k, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness_batch(pk_g, h, _p(wl), m, k, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness_batch(pk_shard, h, _p(wl), m, k, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness_batch(pk, h, None, m, k, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness_batch(pk, h, _p(wl), m, k, None, _p(pb)),
            L.b200_pinocchio_prove_witness_batch(pk, h, _p(wl), m, k, _p(g1), None),
            L.b200_pinocchio_prove_witness_batch(pk, h, _p(wl), m + 1, k, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness_batch(pk, small.r1cs.handle, _p(wl), m, k, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness_batch_device(pk, h, W, m, 0, O, None),
            L.b200_pinocchio_prove_witness_batch_device(pk_g, h, W, m, k, O, None),
            L.b200_pinocchio_prove_witness_batch_device(pk_shard, h, W, m, k, O, None),
            L.b200_pinocchio_prove_witness_batch_device(pk, h, None, m, k, O, None),
            L.b200_pinocchio_prove_witness_batch_device(pk, h, W, m, k, None, None),
            L.b200_pinocchio_prove_witness_batch_device(pk, h, W, m - 1, k, O, None),
            L.b200_pinocchio_prove_witness_batch_device(pk, h, W, m, too_many, O, None),
            L.b200_pinocchio_prove_witness_batch_device(pk, h, W, m, 1 << 40, O, None),
        ]
        assert bad == [EINVAL] * len(bad), bad
        assert pk_bytes(L, pk) == before
        want = [affine(witness_device(L, pk, h, limbs(w))) for w in wits]
        w_bad = wl.copy()
        w_bad[2 * m + 7] = limbs([R])[0]
        g1[:], pb[:] = 7, 9
        assert L.b200_pinocchio_prove_witness_batch(pk, h, _p(w_bad), m, k, _p(g1), _p(pb)) == ERANGE
        assert (g1 == 7).all() and (pb == 9).all()
        assert [affine(p) for p in batch_host(L, pk, h, wl, m, k)] == want
        # the device entry reads the entry as 0 and no call reports it
        w_zero = [list(w) for w in wits]
        w_zero[2][7] = 0
        got = run_device_batch(L, pk, h, w_bad, m, k)
        assert affine(got[2]) == affine(witness_device(L, pk, h, limbs(w_zero[2])))
        assert [affine(p) for i, p in enumerate(got) if i != 2] == [a for i, a in enumerate(want) if i != 2]
        assert [affine(p) for p in batch_host(L, pk, h, wl, m, k)] == want
    finally:
        for key in (pk, pk_g, pk_shard):
            check(L.b200_pk_free(key))
        groth.r1cs.free()
