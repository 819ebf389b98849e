"""GPU: witness-fed Groth16 proving (include/b200snark.h: b200_groth16_prove_witness, b200_groth16_prove_witness_device).

The quotient comes from the resident sparse R1CS on the device, on the key's prove context and with that context's own
R1CS workspace.  Every proof is checked against the known discrete logs of CircuitGroth16 (groth16.GenerateProofs,
groth16.go:225-278, in the exponent) or against the Go binary's goldens, and verified under the real Vk."""
import ctypes
import json
import os
import threading

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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
    """CircuitGroth16 of n constraints, minted once per module (m = n + 2, len(Z) = n + 1: the h-direct branch)."""
    from gosnark_b200.synthetic import CircuitGroth16
    if n not in _circuits:
        _circuits[n] = CircuitGroth16(n=n)
    return _circuits[n]


def to_dev(arr):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def limbs(v):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs([v])


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


def host_prove(L, pk, w, px, r, s):
    from gosnark_b200._lib import check, ptr
    pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
    check(L.b200_groth16_prove(pk, ptr(w), w.shape[0], ptr(px), px.shape[0], ptr(limbs(r)), ptr(limbs(s)), ptr(pa), ptr(pb),
                               ptr(pc)))
    return split(np.concatenate([pa, pc, pb]))


def host_prove_witness(L, pk, r1cs, w, r, s):
    from gosnark_b200._lib import check, ptr
    pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
    check(L.b200_groth16_prove_witness(pk, r1cs, ptr(w), w.shape[0], ptr(limbs(r)), ptr(limbs(s)), ptr(pa), ptr(pb), ptr(pc)))
    return split(np.concatenate([pa, pc, pb]))


def witness_device(L, pk, r1cs, d_w, m, r, s, d_out, stream=None):
    from gosnark_b200._lib import ptr
    return L.b200_groth16_prove_witness_device(pk, r1cs, d_w.data_ptr(), m, ptr(limbs(r)), ptr(limbs(s)), d_out.data_ptr(),
                                               None if stream is None else stream.cuda_stream)


def load_pk(L, syn, ctx=0, acc=0, rank=0, world=1):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    try:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, ctx))
        check(L.b200_config(_lib.CFG_ACC_MODE, acc))
        return syn.load_pk(rank, world)
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))
        check(L.b200_config(_lib.CFG_ACC_MODE, 0))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n,acc", [(1 << 6, 0), ((1 << 12) + 2, 1), ((1 << 12) + 2, 2), (1 << 16, 0)],
                         ids=["64", "4098-affine", "4098-xyzz", "65536"])
def test_entry_points_agree(L, n, acc):
    """b200_groth16_prove_witness_device (library stream and a torch side stream), b200_groth16_prove_witness and
    b200_groth16_prove with px give the same affine proof, which is the known-discrete-log proof and verifies."""
    import torch
    from gosnark_b200._lib import check
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
    syn = circuit(n)
    pk = load_pk(L, syn, acc=acc)
    try:
        exp = expected(syn.expected_dlogs())
        h = syn.r1cs.handle
        got = {"px": host_prove(L, pk, syn.w, syn.px, syn.r, syn.s),
               "witness": host_prove_witness(L, pk, h, syn.w, syn.r, syn.s)}
        d_w = to_dev(syn.w)
        for name, stream in (("device", None), ("device-side-stream", torch.cuda.Stream())):
            d_out = torch.full((48,), -1, dtype=torch.int64, device="cuda")
            check(witness_device(L, pk, h, d_w, syn.m, syn.r, syn.s, d_out, stream))
            torch.cuda.synchronize()          # the library's stream is not ordered with any torch stream
            got[name] = split(d_out.cpu().numpy().view(np.uint64))
        for name, p in got.items():
            assert affine(p) == exp, name
        pa, pb, pc = got["device"]
        assert syn.verify(_flatten_g1([pa]), _flatten_g2([pb]), _flatten_g1([pc]))
    finally:
        check(L.b200_pk_free(pk))


def _load_golden(golden_dir, name):
    with open(os.path.join(golden_dir, f"gobin_{name}.json")) as f:
        return json.load(f)


def _groth_pk(setup):
    t3 = tuple
    g2t = lambda p: tuple(tuple(c) for c in p)
    pk = setup["Pk"]
    return {"Z": pk["Z"], "BACDelta": [t3(p) for p in pk["BACDelta"]], "PowersTauDelta": [t3(p) for p in pk["PowersTauDelta"]],
            "G1": {"Alpha": t3(pk["G1"]["Alpha"]), "Beta": t3(pk["G1"]["Beta"]), "Delta": t3(pk["G1"]["Delta"]),
                   "At": [t3(p) for p in pk["G1"]["At"]], "BACGamma": [t3(p) for p in pk["G1"]["BACGamma"]]},
            "G2": {"Beta": g2t(pk["G2"]["Beta"]), "Delta": g2t(pk["G2"]["Delta"]),
                   "BACGamma": [g2t(p) for p in pk["G2"]["BACGamma"]]}}


def _groth_vk(setup):
    vk = setup["Vk"]
    g2t = lambda p: tuple(tuple(c) for c in p)
    return {"IC": [tuple(p) for p in vk["IC"]], "G1": {"Alpha": tuple(vk["G1"]["Alpha"])},
            "G2": {k: g2t(vk["G2"][k]) for k in ("Beta", "Gamma", "Delta")}}


@pytest.mark.parametrize("name", ["x3x5", "chain21", "mul"])
def test_golden_circuits(L, golden_dir, name):
    """The Go binary's circuits: x3x5 and chain21 have m = n + 1 and len(Z) = n, so the witness entries take the
    short-Z quotient (mul, len(Z) = n + 1, the h-direct one).  The device witness entry, the host witness entry
    (DeviceProvingKey.prove_witness_limbs) and b200_groth16_prove with the golden px give the same proof for the same
    r, s, and it verifies under the golden Vk."""
    import torch
    from gosnark_b200 import groth16
    from gosnark_b200._lib import check, ints_to_limbs
    from gosnark_b200.bn128 import reduce_scalar
    from gosnark_b200.r1csqap import SparseR1CS
    g = _load_golden(golden_dir, name)
    cc = g["compiledcircuit"]
    a, b, c = cc["R1CS"]["A"], cc["R1CS"]["B"], cc["R1CS"]["C"]
    n, m = len(a), len(a[0])
    assert m == cc["NVars"]
    sp = SparseR1CS(n, m, (a, b, c))
    dpk = groth16.DeviceProvingKey(_groth_pk(g["groth16_setup"]), m, cc["NPublic"])
    assert (len(g["groth16_setup"]["Pk"]["Z"]) == n + 1) == (name == "mul")
    try:
        r, s = 0x1234567890ABCDEF << 100, 0xFEDCBA0987654321 << 90
        w = ints_to_limbs([reduce_scalar(x) for x in g["witness"]])
        px = ints_to_limbs([int(x) % R for x in g["px"]])
        ref = dpk.prove_limbs(w, px, r, s)
        host = dpk.prove_witness_limbs(sp, w, r, s)
        d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
        check(witness_device(L, dpk.handle, sp.handle, to_dev(w), m, r, s, d_out))
        torch.cuda.synchronize()
        dev = dict(zip(("PiA", "PiB", "PiC"), split(d_out.cpu().numpy().view(np.uint64))))
        for k, G in (("PiA", G1), ("PiB", G2), ("PiC", G1)):
            assert G.affine(host[k]) == G.affine(ref[k]), k
            assert G.affine(dev[k]) == G.affine(ref[k]), k
        assert groth16.VerifyProof(_groth_vk(g["groth16_setup"]), dev, g["public"])
    finally:
        dpk.free()
        sp.free()


def _two_context_setup(L, n):
    """Keys of contexts 0 and 1 of one CircuitGroth16 sharing ONE R1CS handle, and two satisfying witnesses."""
    from gosnark_b200._lib import ints_to_limbs
    from gosnark_b200.synthetic import SyntheticCircuit
    syn = circuit(n)
    pks = [load_pk(L, syn, ctx=k) for k in range(2)]
    wits = [syn.circuit.witness, SyntheticCircuit(n, seed=0xD1FF).witness]
    assert wits[0] != wits[1]
    return syn, pks, wits, [ints_to_limbs(w) for w in wits]


@pytest.mark.timeout(900)
def test_two_contexts_in_flight_share_one_r1cs(L):
    """Four rounds on two streams with no host synchronisation: round j proves on the context-k key from witness
    (j + k) mod 2 with its own r, s.  Different witnesses per context make a workspace race visible: with one shared
    witness both contexts would write identical values.  Both streams wait behind a gate kernel while all eight proofs are
    enqueued, so the two contexts' QAP front ends start together instead of being spaced out by the host; the gate is
    still closed when the last call returns (no call waited for the device).  Every proof matches its own expectation."""
    import torch
    from gosnark_b200._lib import check
    syn, pks, wits, wl = _two_context_setup(L, 1 << 14)
    try:
        d_w = [to_dev(x) for x in wl]
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        rounds = 4
        outs = {(j, k): torch.zeros(48, dtype=torch.int64, device="cuda") for j in range(rounds) for k in range(2)}
        rs = {(j, k): ((syn.r + 31 * (2 * j + k)) % R, (syn.s + 37 * (2 * j + k)) % R) for j in range(rounds) for k in range(2)}
        for k in range(2):      # the first call on each (R1CS, context) pair builds the domains and workspaces
            check(witness_device(L, pks[k], syn.r1cs.handle, d_w[k], syn.m, *rs[(0, k)], outs[(0, k)], streams[k]))
        torch.cuda.synchronize()
        gate = torch.cuda.Stream()
        with torch.cuda.stream(gate):
            torch.cuda._sleep(400_000_000)     # ~0.2 s of SM cycles
        opened = torch.cuda.Event()
        opened.record(gate)
        for st in streams:
            st.wait_event(opened)
        for j in range(rounds):
            for k in range(2):
                check(witness_device(L, pks[k], syn.r1cs.handle, d_w[(j + k) % 2], syn.m, *rs[(j, k)], outs[(j, k)], streams[k]))
        assert not opened.query(), "an enqueue waited for the device"
        torch.cuda.synchronize()
        for (j, k), d in outs.items():
            exp = expected(syn.expected_dlogs(wits[(j + k) % 2], *rs[(j, k)]))
            assert affine(split(d.cpu().numpy().view(np.uint64))) == exp, (j, k)
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_two_host_threads_share_one_r1cs(L):
    """b200_groth16_prove_witness from two host threads, thread k on the context-k key, both on one R1CS handle, each
    round with another witness and r, s: the waits run with the library mutex released, so the proofs overlap."""
    from gosnark_b200._lib import check
    syn, pks, wits, wl = _two_context_setup(L, 1 << 13)
    rounds = 3
    results, errs = {}, []

    def worker(k):
        try:
            for j in range(rounds):
                r_, s_ = (syn.r + 101 * (2 * j + k)) % R, (syn.s + 103 * (2 * j + k)) % R
                results[(k, j)] = (r_, s_, host_prove_witness(L, pks[k], syn.r1cs.handle, wl[(j + k) % 2], r_, s_))
        except Exception as e:   # noqa: BLE001 - reported below
            errs.append(e)

    try:
        ths = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        assert not errs, errs
        assert len(results) == 2 * rounds
        for (k, j), (r_, s_, p) in results.items():
            assert affine(p) == expected(syn.expected_dlogs(wits[(j + k) % 2], r_, s_)), (k, j)
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


def _launches(L, fn):
    from gosnark_b200._lib import check
    out = (ctypes.c_double * 8)()
    check(L.b200_profile_read(out))          # synchronises and resets the counter
    fn()
    check(L.b200_profile_read(out))
    return int(out[6])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_emulated_on_one_gpu(L, world):
    """Every rank calls b200_groth16_prove_witness_device, then b200_groth16_finalize_device sums the records: the
    unsharded proof and the expectation.  Under b200_profile's launch counter, a rank that holds no PowersTauDelta index
    (needs_px 0) issues exactly the launches of b200_groth16_prove_device on its key: no QAP kernel.  A rank that holds
    some runs the whole QAP front end in place of the division, so its count differs from its px-fed proof's by exactly
    what it does on the unsharded key (the division of a px-fed proof issues more launches than the h-direct front end at
    this size, so the difference is negative).  Without a communicator the host witness entry refuses a sharded key."""
    import torch
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check, ptr
    syn = circuit(1 << 10)
    h = syn.r1cs.handle
    m, npx = syn.m, syn.px.shape[0]
    d_w, d_px = to_dev(syn.w), to_dev(syn.px)
    rr, ss = limbs(syn.r), limbs(syn.s)
    pk1 = load_pk(L, syn)
    pks = [load_pk(L, syn, rank=rk, world=world) for rk in range(world)]
    try:
        d_single = torch.zeros(48, dtype=torch.int64, device="cuda")
        check(witness_device(L, pk1, h, d_w, m, syn.r, syn.s, d_single))
        parts = torch.zeros(128 * world, dtype=torch.int64, device="cuda")
        for rk, pk in enumerate(pks):
            check(witness_device(L, pk, h, d_w, m, syn.r, syn.s, parts[128 * rk:]))
        d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
        check(L.b200_groth16_finalize_device(pks[0], parts.data_ptr(), world, ptr(rr), ptr(ss), d_out.data_ptr(), None))
        torch.cuda.synchronize()
        check(L.b200_profile_read((ctypes.c_double * 8)()))
        exp = expected(syn.expected_dlogs())
        assert affine(split(d_single.cpu().numpy().view(np.uint64))) == exp
        assert affine(split(d_out.cpu().numpy().view(np.uint64))) == exp
        scratch = torch.zeros(128, dtype=torch.int64, device="cuda")

        def launch_delta(pk):
            """launches of the witness-fed proof minus those of the px-fed one, on key pk"""
            base = _launches(L, lambda: check(L.b200_groth16_prove_device(pk, d_w.data_ptr(), m, d_px.data_ptr(), npx, ptr(rr),
                                                                          ptr(ss), scratch.data_ptr(), None)))
            return _launches(L, lambda: check(witness_device(L, pk, h, d_w, m, syn.r, syn.s, scratch))) - base
        qap_delta = launch_delta(pk1)
        assert qap_delta != 0
        needs, deltas = [], []
        for pk in pks:
            info = np.zeros(12, dtype=np.uint64)
            check(L.b200_groth16_shard_info(pk, ptr(info)))
            needs.append(int(info[8]))
            deltas.append(launch_delta(pk))
        assert deltas == [qap_delta if nd else 0 for nd in needs], (needs, deltas, qap_delta)
        assert any(needs) and not all(needs), needs
        with pytest.raises(_lib.B200Error) as ei:
            host_prove_witness(L, pks[-1], h, syn.w, syn.r, syn.s)
        assert ei.value.code == EINVAL and "b200_groth16_prove_witness_device" in str(ei.value)
    finally:
        for pk in pks + [pk1]:
            check(L.b200_pk_free(pk))


def _comm_worker(rank, world, uid, n, ret):
    import sys
    sys.path.insert(0, ROOT)
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check, ptr
    from gosnark_b200.synthetic import CircuitGroth16
    try:
        _lib.init(rank)
        L = _lib.lib()
        syn = CircuitGroth16(n=n)
        pk = syn.load_pk(rank, world)
        check(L.b200_comm_init(ptr(np.frombuffer(uid, dtype=np.uint8).copy()), rank, world))
        p = host_prove_witness(L, pk, syn.r1cs.handle, syn.w, syn.r, syn.s)
        ret.put((rank, affine(p) == expected(syn.expected_dlogs())))
        check(L.b200_comm_destroy())
    except Exception as e:   # noqa: BLE001 - reported to the parent
        ret.put((rank, repr(e)))


@pytest.mark.timeout(900)
def test_sharded_host_entry_with_communicator(L):
    """SPMD over a real NCCL communicator, one process per GPU: b200_groth16_prove_witness on a sharded key returns the
    whole proof on every rank.  Needs at least two visible GPUs."""
    import torch
    import torch.multiprocessing as mp
    from gosnark_b200._lib import check, ptr
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs at least two GPUs")
    uid = np.zeros(128, dtype=np.uint8)
    check(L.b200_comm_unique_id(ptr(uid)))
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_comm_worker, args=(rk, world, uid.tobytes(), 1 << 10, ret)) for rk in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
    got = dict(ret.get(timeout=5) for _ in range(world))
    assert all(v is True for v in got.values()), got
    assert all(p.exitcode == 0 for p in procs)


@pytest.mark.timeout(600)
def test_argument_errors_and_out_of_range_witness(L):
    """Bad handles, null pointers, nw != m, an R1CS whose m differs from the key's, and r or s >= r return the documented
    codes and the key still proves.  A witness entry >= r on the device entry is read as 0 and reported by nobody: the
    next b200_groth16_prove and b200_g1_msm succeed."""
    import torch
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    from gosnark_b200.r1csqap import SparseR1CS
    from gosnark_b200.synthetic import SyntheticCircuit, mint_points, rand_limbs
    syn = circuit(1 << 6)
    pk = load_pk(L, syn)
    h, m = syn.r1cs.handle, syn.m
    other = SyntheticCircuit(syn.n + 1)
    sp_other = SparseR1CS(other.n, other.m, other.csr)
    d_w = to_dev(syn.w)
    d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
    rr, ss, big = limbs(syn.r), limbs(syn.s), limbs(R)
    try:
        calls = {
            "bad key": (0, h, d_w.data_ptr(), m, rr, ss, d_out.data_ptr(), EINVAL),
            "bad r1cs": (pk, 0xDEAD, d_w.data_ptr(), m, rr, ss, d_out.data_ptr(), EINVAL),
            "null witness": (pk, h, None, m, rr, ss, d_out.data_ptr(), EINVAL),
            "null out": (pk, h, d_w.data_ptr(), m, rr, ss, None, EINVAL),
            "null r": (pk, h, d_w.data_ptr(), m, None, ss, d_out.data_ptr(), EINVAL),
            "nw != m": (pk, h, d_w.data_ptr(), m - 1, rr, ss, d_out.data_ptr(), EINVAL),
            "r1cs m != key m": (pk, sp_other.handle, d_w.data_ptr(), m, rr, ss, d_out.data_ptr(), EINVAL),
            "r1cs m, nw != key m": (pk, sp_other.handle, d_w.data_ptr(), other.m, rr, ss, d_out.data_ptr(), EINVAL),
            "r >= r": (pk, h, d_w.data_ptr(), m, big, ss, d_out.data_ptr(), ERANGE),
            "s >= r": (pk, h, d_w.data_ptr(), m, rr, big, d_out.data_ptr(), ERANGE),
        }
        for what, (k, r1, dw, nw, r_, s_, out, code) in calls.items():
            rc = L.b200_groth16_prove_witness_device(k, r1, dw, nw, None if r_ is None else ptr(r_), ptr(s_), out, None)
            assert rc == code, what
        pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
        for what, (k, r1, w_, nw, r_, s_, code) in {
                "bad key": (0, h, syn.w, m, rr, ss, EINVAL), "bad r1cs": (pk, 0xDEAD, syn.w, m, rr, ss, EINVAL),
                "nw != m": (pk, h, syn.w, m - 1, rr, ss, EINVAL), "r1cs m != key m": (pk, sp_other.handle, syn.w, m, rr, ss, EINVAL),
                "r >= r": (pk, h, syn.w, m, big, ss, ERANGE), "s >= r": (pk, h, syn.w, m, rr, big, ERANGE)}.items():
            rc = L.b200_groth16_prove_witness(k, r1, ptr(w_), nw, ptr(r_), ptr(s_), ptr(pa), ptr(pb), ptr(pc))
            assert rc == code, what
        assert L.b200_groth16_prove_witness(pk, h, None, m, ptr(rr), ptr(ss), ptr(pa), ptr(pb), ptr(pc)) == EINVAL
        exp = expected(syn.expected_dlogs())
        check(witness_device(L, pk, h, d_w, m, syn.r, syn.s, d_out))
        torch.cuda.synchronize()
        assert affine(split(d_out.cpu().numpy().view(np.uint64))) == exp
        # an out-of-range witness entry on the device entry: the key's own error word, never reported
        bad = syn.w.copy()
        bad[syn.npublic + 3] = ints_to_limbs([R])[0]
        check(witness_device(L, pk, h, to_dev(bad), m, syn.r, syn.s, d_out))
        torch.cuda.synchronize()
        assert affine(host_prove(L, pk, syn.w, syn.px, syn.r, syn.s)) == exp
        assert affine(host_prove_witness(L, pk, h, syn.w, syn.r, syn.s)) == exp
        ks = rand_limbs(4, 77)
        bases = _lib._h(0)
        check(L.b200_g1_bases_load(ptr(mint_points(1, ks)), 4, 0, bases))
        sc = rand_limbs(4, 78)
        out = np.zeros(12, np.uint64)
        check(L.b200_g1_msm(bases.value, ptr(sc), 4, ptr(out)))
        check(L.b200_bases_free(bases.value))
    finally:
        check(L.b200_pk_free(pk))
        sp_other.free()
