"""GPU: witness-fed and device-resident Pinocchio proving (include/b200snark.h: b200_pinocchio_prove_device,
b200_pinocchio_prove_witness, b200_pinocchio_prove_witness_device) on synthetic.CircuitPinocchio — a real key and Vk with
known discrete logs — and on the Go binary's circuits.  Proofs are compared on affine coordinates, element by element."""
import ctypes
import json
import os
import random
import shutil
import subprocess
import tempfile
import threading

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G1, G2 = o.BN.G1, o.BN.G2
R = o.R
ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")
EINVAL, ERANGE = -3, -4


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


_circuits = {}


def circuit(n):
    """CircuitPinocchio of n constraints (len(Z) = n + 1: the h-direct branch), minted once per module."""
    from gosnark_b200.synthetic import CircuitPinocchio
    if n not in _circuits:
        _circuits[n] = CircuitPinocchio(n)
    return _circuits[n]


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


def split(words):
    """108 u64 (seven G1 points, then PiB) -> proof dict."""
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    proof = dict(zip(ORDER, _unflatten_g1(words[:84])))
    proof["PiB"] = _unflatten_g2(words[84:108])[0]
    return proof


def affine(proof):
    return tuple(G1.affine(proof[k]) for k in ORDER) + (G2.affine(proof["PiB"]),)


def expected(dlogs):
    return tuple(G1.affine(G1.mul_scalar(G1.G, dlogs[k])) for k in ORDER) + (G2.affine(G2.mul_scalar(G2.G, dlogs["PiB"])),)


def px_fed(L, pk, w, px):
    from gosnark_b200._lib import check
    g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
    check(L.b200_pinocchio_prove(pk, _p(w), w.shape[0], _p(px), px.shape[0], _p(g1), _p(pb)))
    return split(np.concatenate([g1, pb]))


def px_fed_device(L, pk, w, px, stream=None):
    import torch
    from gosnark_b200._lib import check
    d_w, d_px = to_dev(w), to_dev(px)
    d_out = torch.full((108,), -1, dtype=torch.int64, device="cuda")
    check(L.b200_pinocchio_prove_device(pk, d_w.data_ptr(), w.shape[0], d_px.data_ptr(), px.shape[0], d_out.data_ptr(),
                                        None if stream is None else stream.cuda_stream))
    torch.cuda.synchronize()
    return split(d_out.cpu().numpy().view(np.uint64))


def witness_host(L, pk, r1cs, w):
    from gosnark_b200._lib import check
    g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
    check(L.b200_pinocchio_prove_witness(pk, r1cs, _p(w), w.shape[0], _p(g1), _p(pb)))
    return split(np.concatenate([g1, pb]))


def witness_device(L, pk, r1cs, w, stream=None):
    import torch
    from gosnark_b200._lib import check
    d_w = to_dev(w)
    d_out = torch.full((108,), -1, dtype=torch.int64, device="cuda")
    check(L.b200_pinocchio_prove_witness_device(pk, r1cs, d_w.data_ptr(), w.shape[0], d_out.data_ptr(),
                                                None if stream is None else stream.cuda_stream))
    torch.cuda.synchronize()
    return split(d_out.cpu().numpy().view(np.uint64))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("acc", [1, 2], ids=["affine", "xyzz"])
@pytest.mark.parametrize("n", [1 << 12, (1 << 12) + 2, 1 << 16])
def test_four_entries_agree_and_verify(L, n, acc):
    """Witness-fed host == witness-fed device == px-fed device == b200_pinocchio_prove, equal to the known-discrete-log
    proof, accepted under the real Vk; a second witness on the same key (reused scratch) as well."""
    import torch
    from gosnark_b200._lib import check
    from gosnark_b200.synthetic import SyntheticCircuit
    syn = circuit(n)
    pk = load_pk(L, syn, acc=acc)
    try:
        other = SyntheticCircuit(n, seed=0x5EED0202)
        for w, wit, pub in ((syn.w, None, None), (limbs(other.witness), other.witness, other.public_signals)):
            px = syn.px_of(w)
            want = expected(syn.expected_dlogs(wit))
            runs = {"witness-host": witness_host(L, pk, syn.r1cs.handle, w),
                    "witness-device": witness_device(L, pk, syn.r1cs.handle, w),
                    "witness-device-side-stream": witness_device(L, pk, syn.r1cs.handle, w, torch.cuda.Stream()),
                    "px-device": px_fed_device(L, pk, w, px),
                    "px-host": px_fed(L, pk, w, px)}
            for name, proof in runs.items():
                assert affine(proof) == want, name
            assert syn.verify(runs["witness-device"], pub)
    finally:
        check(L.b200_pk_free(pk))


def _golden(golden_dir, name):
    with open(os.path.join(golden_dir, f"gobin_{name}.json")) as f:
        return json.load(f)


def pinocchio_pk(setup):
    t3 = tuple
    pk = {k: [t3(p) for p in setup["Pk"][k]] for k in ("A", "C", "Kp", "Ap", "Bp", "Cp")}
    pk["B"] = [tuple(tuple(c) for c in p) for p in setup["Pk"]["B"]]
    pk["Z"] = setup["Pk"]["Z"]
    pk["G1T"] = [t3(p) for p in setup["G1T"]]
    return pk


def go_verify(g, proof):
    """The reference's own Go code on our proof (cli/main.go verify); None when the binary is not staged."""
    binary = os.path.join(ROOT, "oracle", "_ref", "go-snark-cli")
    if not os.path.exists(binary):
        return None
    d = tempfile.mkdtemp(prefix="gsv_")
    try:
        b = os.path.join(d, "gsc")
        shutil.copy(binary, b)
        os.chmod(b, 0o755)
        pj = {k: (list(v) if k != "PiB" else [list(c) for c in v]) for k, v in proof.items()}
        for fname, obj in (("trustedsetup.json", g["pinocchio_setup"]), ("compiledcircuit.json", g["compiledcircuit"]),
                           ("publicInputs.json", g["public"]), ("proofs.json", pj)):
            with open(os.path.join(d, fname), "w") as f:
                json.dump(obj, f)
        p = subprocess.run([b, "verify"], cwd=d, capture_output=True, text=True, timeout=120)
        return p.stdout + p.stderr
    finally:
        shutil.rmtree(d)


@pytest.mark.parametrize("name", ["x3x5", "chain21", "mul"])
def test_go_binary_circuits(L, golden_dir, name):
    """The Go binary's circuits: the witness-fed proof equals the binary's proofs.json, and the binary verifies it.  x3x5
    and chain21 (len(Z) = n) take the short-Z quotient on the device, mul the h-direct one."""
    from gosnark_b200 import snark
    from gosnark_b200._lib import ints_to_limbs
    from gosnark_b200.bn128 import reduce_scalar
    from gosnark_b200.r1csqap import SparseR1CS
    g = _golden(golden_dir, name)
    cc = g["compiledcircuit"]
    a, b, c = cc["R1CS"]["A"], cc["R1CS"]["B"], cc["R1CS"]["C"]
    n, m = len(a), len(a[0])
    assert (len(g["pinocchio_setup"]["Pk"]["Z"]) == n + 1) == (name == "mul")
    sp = SparseR1CS(n, m, (a, b, c))
    dpk = snark.DeviceProvingKey(pinocchio_pk(g["pinocchio_setup"]), m, cc["NPublic"])
    try:
        w = ints_to_limbs([reduce_scalar(x) for x in g["witness"]])
        proof = dpk.prove_witness_limbs(sp, w)
        ref = g["pinocchio_proofs"]
        for k in ORDER:
            assert G1.affine(proof[k]) == G1.affine(tuple(ref[k])), k
        assert G2.affine(proof["PiB"]) == G2.affine(tuple(tuple(c) for c in ref["PiB"]))
        assert affine(witness_device(L, dpk.handle, sp.handle, w)) == affine(proof)
        out = go_verify(g, proof)
        if out is not None:
            assert "Proofs verified" in out and "❌" not in out, out
    finally:
        dpk.free()
        sp.free()


def unsatisfied(syn, how):
    """A witness of syn's circuit that breaks one row's signal, or every entry random (ints)."""
    w = list(syn.circuit.witness)
    if how == "one":
        w[syn.n // 2 + 2] = (w[syn.n // 2 + 2] + 1) % R
        return w
    rng = random.Random(syn.n)
    return [1] + [rng.randrange(R) for _ in range(syn.m - 1)]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("how", ["one", "every"])
@pytest.mark.parametrize("n", [1 << 10, (1 << 12) + 2])
def test_unsatisfied_witness_gets_the_px_fed_proof(L, n, how):
    """The quotient drops the remainder: an unsatisfied witness gets the proof b200_pinocchio_prove gives for it and its
    px, and the proof is refused."""
    from gosnark_b200._lib import check
    syn = circuit(n)
    pk = load_pk(L, syn)
    try:
        wi = unsatisfied(syn, how)
        w = limbs(wi)
        ref = px_fed(L, pk, w, syn.px_of(w))
        assert affine(witness_device(L, pk, syn.r1cs.handle, w)) == affine(ref)
        got = witness_host(L, pk, syn.r1cs.handle, w)
        assert affine(got) == affine(ref)
        assert not syn.verify(got, [wi[1]])
    finally:
        check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_two_proofs_in_flight(L):
    """Keys of contexts 0 and 1 on one R1CS handle: b200_pinocchio_prove_witness_device on two streams, interleaved for
    several rounds with no host synchronisation after the first call per context; then the host entry from two threads."""
    import torch
    from gosnark_b200._lib import check
    from gosnark_b200.synthetic import SyntheticCircuit
    n = 1 << 12
    syn = circuit(n)
    pks = [load_pk(L, syn, ctx=c) for c in range(2)]
    try:
        cs = [SyntheticCircuit(n, seed=0xF11 + j) for j in range(4)]
        want = [expected(syn.expected_dlogs(c.witness)) for c in cs]
        d_w = [to_dev(limbs(c.witness)) for c in cs]
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        for c in range(2):      # the first call per (R1CS, context) builds its workspace and may synchronise
            d = torch.zeros(108, dtype=torch.int64, device="cuda")
            check(L.b200_pinocchio_prove_witness_device(pks[c], syn.r1cs.handle, d_w[c].data_ptr(), syn.m, d.data_ptr(),
                                                        streams[c].cuda_stream))
        torch.cuda.synchronize()
        outs = {}
        for j in range(4):
            for c in range(2):
                wi = (j + 2 * c) % 4
                outs[(j, c, wi)] = torch.zeros(108, dtype=torch.int64, device="cuda")
                check(L.b200_pinocchio_prove_witness_device(pks[c], syn.r1cs.handle, d_w[wi].data_ptr(), syn.m,
                                                            outs[(j, c, wi)].data_ptr(), streams[c].cuda_stream))
        torch.cuda.synchronize()
        for (j, c, wi), d in outs.items():
            assert affine(split(d.cpu().numpy().view(np.uint64))) == want[wi], (j, c)
        results, errs = {}, []

        def worker(c):
            try:
                for j in range(3):
                    wi = (j + c) % 4
                    results[(c, j, wi)] = witness_host(L, pks[c], syn.r1cs.handle, limbs(cs[wi].witness))
            except Exception as e:   # noqa: BLE001 - reported below
                errs.append(e)
        ths = [threading.Thread(target=worker, args=(c,)) for c in range(2)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        assert not errs, errs
        for (c, j, wi), proof in results.items():
            assert affine(proof) == want[wi], (c, j)
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_pinocchio_and_groth16_keys_share_a_context_workspace(L):
    """A Pinocchio key and a Groth16 key of one context proving alternately from ONE R1CS handle (they share the
    context's workspace on it): every proof equals its known-discrete-log expectation."""
    import torch
    from gosnark_b200._lib import check
    from gosnark_b200.synthetic import CircuitGroth16
    n = 1 << 12
    syn = circuit(n)
    groth = CircuitGroth16(n=n)
    pk_p = load_pk(L, syn)
    pk_g = groth.load_pk()
    try:
        d_w = to_dev(groth.w)
        assert groth.m == syn.m
        for _ in range(3):
            assert affine(witness_device(L, pk_p, syn.r1cs.handle, syn.w)) == expected(syn.expected_dlogs())
            d = torch.zeros(48, dtype=torch.int64, device="cuda")
            check(L.b200_groth16_prove_witness_device(pk_g, syn.r1cs.handle, d_w.data_ptr(), groth.m, _p(limbs([groth.r])),
                                                      _p(limbs([groth.s])), d.data_ptr(), None))
            torch.cuda.synchronize()
            from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
            raw = d.cpu().numpy().view(np.uint64)
            pa, pc = _unflatten_g1(raw[:24])
            ea, eb, ec = groth.expected_dlogs()
            assert G1.affine(pa) == G1.affine(G1.mul_scalar(G1.G, ea))
            assert G2.affine(_unflatten_g2(raw[24:48])[0]) == G2.affine(G2.mul_scalar(G2.G, eb))
            assert G1.affine(pc) == G1.affine(G1.mul_scalar(G1.G, ec))
    finally:
        check(L.b200_pk_free(pk_p))
        check(L.b200_pk_free(pk_g))
        groth.r1cs.free()


def _launches(L, fn):
    from gosnark_b200._lib import check
    out = (ctypes.c_double * 8)()
    check(L.b200_profile_read(out))          # synchronises and resets the counter
    fn()
    check(L.b200_profile_read(out))
    return int(out[6])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_records(L, world):
    """Whole MSMs dealt to `world` ranks, emulated on one GPU: the records b200_pinocchio_prove_witness_device leaves on
    keys without a communicator, summed by b200_pinocchio_finalize_records, are the unsharded proof; so are those of
    b200_pinocchio_prove_device.  Only the rank that holds G1T runs the QAP front end: every other rank issues fewer
    launches.  The host entry refuses a sharded key without a communicator."""
    import torch
    from gosnark_b200._lib import check
    syn = circuit(1 << 12)
    pks = [load_pk(L, syn, acc=1, rank=rk, world=world) for rk in range(world)]
    try:
        d_w, d_px = to_dev(syn.w), to_dev(syn.px)
        want = expected(syn.expected_dlogs())
        counts = []
        for entry in ("witness", "px"):
            recs = torch.zeros(256 * world, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            for rk, pk in enumerate(pks):
                if entry == "witness":
                    run = lambda: check(L.b200_pinocchio_prove_witness_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m,
                                                                              recs[256 * rk:].data_ptr(), None))
                    run()                                       # the first call builds the workspace
                    counts.append(_launches(L, run))
                else:
                    check(L.b200_pinocchio_prove_device(pk, d_w.data_ptr(), syn.m, d_px.data_ptr(), syn.px.shape[0],
                                                        recs[256 * rk:].data_ptr(), None))
            torch.cuda.synchronize()
            g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
            check(L.b200_pinocchio_finalize_records(recs.data_ptr(), world, _p(g1), _p(pb)))
            assert affine(split(np.concatenate([g1, pb]))) == want, entry
        # the owner of G1T runs the front end and the G1T MSM on top of a share of the other seven
        owner = max(range(world), key=lambda rk: counts[rk])
        scratch = torch.zeros(256, dtype=torch.int64, device="cuda")
        others = [c for rk, c in enumerate(counts) if rk != owner]
        assert all(c < counts[owner] for c in others), counts
        # a rank without G1T issues exactly what its px-fed proof issues: no QAP kernel
        rk = next(r for r in range(world) if r != owner)
        same = _launches(L, lambda: check(L.b200_pinocchio_prove_device(
            pks[rk], d_w.data_ptr(), syn.m, d_px.data_ptr(), syn.px.shape[0], scratch.data_ptr(), None)))
        assert same == counts[rk], (same, counts)
        g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
        assert L.b200_pinocchio_prove_witness(pks[0], syn.r1cs.handle, _p(syn.w), syn.m, _p(g1), _p(pb)) == EINVAL
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


def pk_bytes(L, pk):
    from gosnark_b200._lib import check
    v = ctypes.c_size_t(0)
    check(L.b200_pk_device_bytes(pk, ctypes.byref(v)))
    return v.value


@pytest.mark.timeout(600)
def test_errors(L):
    """Every B200_EINVAL of the three entries leaves b200_pk_device_bytes unchanged; a witness entry >= r gives B200_ERANGE
    on the host entry, leaves the outputs untouched, and the next proof is right; on the device entry it is read as 0 and
    reported by no call; a Groth16 key is refused, and b200_groth16_prove_witness refuses a Pinocchio key."""
    import torch
    from gosnark_b200._lib import check
    from gosnark_b200.synthetic import CircuitGroth16
    syn, small = circuit(1 << 10), circuit(1 << 6)
    groth = CircuitGroth16(n=1 << 6)
    pk, pk_small, pk_g = load_pk(L, syn), load_pk(L, small), groth.load_pk()
    try:
        m, h = syn.m, syn.r1cs.handle
        d_w, d_px = to_dev(syn.w), to_dev(syn.px)
        d_out = torch.zeros(108, dtype=torch.int64, device="cuda")
        g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
        before = pk_bytes(L, pk)
        W, PX, O = d_w.data_ptr(), d_px.data_ptr(), d_out.data_ptr()
        npx = syn.px.shape[0]
        bad = [
            L.b200_pinocchio_prove_witness(pk + 1000, h, _p(syn.w), m, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness(pk, h + 1000, _p(syn.w), m, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness(pk_g, h, _p(syn.w), m, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness(pk, h, None, m, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness(pk, h, _p(syn.w), m, None, _p(pb)),
            L.b200_pinocchio_prove_witness(pk, h, _p(syn.w), m, _p(g1), None),
            L.b200_pinocchio_prove_witness(pk, h, _p(syn.w), m - 1, _p(g1), _p(pb)),
            L.b200_pinocchio_prove_witness(pk, small.r1cs.handle, _p(syn.w), m, _p(g1), _p(pb)),     # R1CS columns != m
            L.b200_pinocchio_prove_witness_device(pk_g, h, W, m, O, None),
            L.b200_pinocchio_prove_witness_device(pk, h, None, m, O, None),
            L.b200_pinocchio_prove_witness_device(pk, h, W, m, None, None),
            L.b200_pinocchio_prove_witness_device(pk, h, W, m + 1, O, None),
            L.b200_pinocchio_prove_device(pk_g, W, m, PX, npx, O, None),
            L.b200_pinocchio_prove_device(pk, None, m, PX, npx, O, None),
            L.b200_pinocchio_prove_device(pk, W, m, None, npx, O, None),
            L.b200_pinocchio_prove_device(pk, W, m, PX, npx, None, None),
            L.b200_pinocchio_prove_device(pk, W, m - 1, PX, npx, O, None),
            L.b200_pinocchio_prove_device(pk, W, m, PX, syn.n, O, None),             # len(px) < len(Z)
            L.b200_pinocchio_prove_device(pk, W, m, PX, 4 * syn.n, O, None),         # len(hx) > len(G1T)
        ]
        assert bad == [EINVAL] * len(bad), bad
        pa, pb2, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
        assert L.b200_groth16_prove_witness(pk, h, _p(syn.w), m, _p(limbs([1])), _p(limbs([2])), _p(pa), _p(pb2), _p(pc)) == EINVAL
        assert pk_bytes(L, pk) == before
        # a witness entry >= r
        w_bad = syn.w.copy()
        w_bad[5] = limbs([R])[0]
        g1[:], pb[:] = 7, 9
        assert L.b200_pinocchio_prove_witness(pk, h, _p(w_bad), m, _p(g1), _p(pb)) == ERANGE
        assert (g1 == 7).all() and (pb == 9).all()
        want = expected(syn.expected_dlogs())
        assert affine(witness_host(L, pk, h, syn.w)) == want
        w_zero = syn.w.copy()
        w_zero[5] = 0
        got = witness_device(L, pk, h, w_bad)                       # read as 0, reported by no call
        assert affine(got) == affine(px_fed(L, pk, w_zero, syn.px_of(w_zero)))
        assert affine(witness_host(L, pk, h, syn.w)) == want
        assert affine(px_fed(L, pk_small, small.w, small.px)) == expected(small.expected_dlogs())
    finally:
        for k in (pk, pk_small, pk_g):
            check(L.b200_pk_free(k))
        groth.r1cs.free()
