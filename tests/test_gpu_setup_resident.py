"""GPU: the trusted setup straight into a device-resident proving key (b200_groth16_setup_pk, b200_pinocchio_setup_pk;
groth16 / snark.GenerateTrustedSetupResident).

The resident key must be the key of the two-step path, GenerateTrustedSetupSparse(...).load_pk(...), for the same toxic
values: the same Vk points, b200_pk_device_bytes and shard info, and the same proofs (px-fed, witness-fed and batched), on
the Go binary's circuits, CircuitGroth16 / CircuitPinocchio and the m = n + 1 variant; under every accumulation mode,
reduced tables, explicit window bits and the second prove context; and per rank of 2, 3 and 8-way shards.  Proofs equal
the known-discrete-log expectation and verify under the returned Vk.  At 2^20 the call must not grow the process's
resident memory by more than a tenth of the two-step path's growth.

Proofs are compared as group elements (affine): their Jacobian words differ from run to run even on one key, because the
MSM's counting sort scatters a bucket's entries with atomics, so the order of additions inside a bucket is not fixed.  That
the two keys' window tables are the same words is checked on the CPU emulation (tests/test_host_setup_key.py)."""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = o.R
G1, G2 = o.BN.G1, o.BN.G2
EINVAL, ERANGE = -3, -4
G16_TOXIC = {"T": 0x1234567890abcdef1234567890abcdef, "Kalpha": 0x1111, "Kbeta": 0x2222222222, "Kgamma": 0x3333,
             "Kdelta": 0x444444}
PIN_TOXIC = {"T": 0x7777777777abcdef12, "Ka": 0x11, "Kb": 0x2222, "Kc": 0x333333, "Kbeta": 0x44, "Kgamma": 0x5555,
             "RhoA": 0x666666, "RhoB": 0x77}
ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")
# groth16_test.go:20-28 circuit (y = x^3 + x + 5): n = 7 constraints, m = 8 signals
A = [[0, 0, 1, 0, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0, 0, 0], [0, 0, 1, 0, 1, 0, 0, 0], [5, 0, 0, 0, 0, 1, 0, 0],
     [0, 0, 0, 0, 0, 0, 1, 0], [0, 1, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0]]
B = [[0, 0, 1, 0, 0, 0, 0, 0], [0, 0, 1, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0],
     [1, 0, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0]]
C = [[0, 0, 0, 1, 0, 0, 0, 0], [0, 0, 0, 0, 1, 0, 0, 0], [0, 0, 0, 0, 0, 1, 0, 0], [0, 0, 0, 0, 0, 0, 1, 0],
     [0, 1, 0, 0, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0, 1, 0], [0, 0, 0, 0, 0, 0, 0, 1]]
W = [1, 35, 3, 9, 27, 30, 35, 1]
RS = [(0x1234567, 0x7654321), (5, 7), (R - 1, 1), (0xabcdef, 0xfedcba)]


@pytest.fixture(scope="module")
def mods():
    from gosnark_b200 import _lib, groth16, r1csqap, snark
    _lib.init()
    return groth16, snark, r1csqap


class Case:
    """A circuit: its sparse R1CS, npublic, a satisfying witness (ints and limbs), px, public signals, and (synthetic
    circuits) the instance that knows the proof's discrete logs."""

    def __init__(self, r1cs, npublic, witness, public, syn=None):
        from gosnark_b200._lib import ints_to_limbs
        self.r1cs, self.npublic, self.syn = r1cs, npublic, syn
        self.witness, self.public = witness, public
        self.w = ints_to_limbs(witness)
        self.px = r1cs.combine_limbs(self.w, want_abc=False)[3]
        self.m = r1cs.m


def golden_case(mods, golden_dir, name):
    r1csqap = mods[2]
    if name == "groth16_test":
        return Case(r1csqap.SparseR1CS(len(A), len(A[0]), (A, B, C)), 1, W, [35])
    with open(os.path.join(golden_dir, f"gobin_{name}.json")) as f:
        d = json.load(f)
    cc = d["compiledcircuit"]
    a, b, c = cc["R1CS"]["A"], cc["R1CS"]["B"], cc["R1CS"]["C"]
    return Case(r1csqap.SparseR1CS(len(a), len(a[0]), (a, b, c)), cc["NPublic"], [int(x) for x in d["witness"]],
                [int(x) for x in d["public"]])


def synthetic_case(proto, n, short_z=False):
    from gosnark_b200.synthetic import CircuitGroth16, CircuitPinocchio
    syn = CircuitGroth16(n=n, mint=False, short_z=short_z) if proto == "g16" else CircuitPinocchio(n, mint=False, short_z=short_z)
    return Case(syn.r1cs, syn.npublic, syn.circuit.witness, syn.circuit.public_signals, syn)


def make_case(mods, golden_dir, proto, name):
    if name.startswith("syn"):
        n = {"syn12": (1 << 12) + 2, "syn16": 1 << 16, "syn12short": (1 << 12) + 2}[name]
        return synthetic_case(proto, n, short_z=name.endswith("short"))
    return golden_case(mods, golden_dir, name)


def toxic_of(proto, case):
    if case.syn is not None:
        return dict(case.syn.toxic)
    return dict(G16_TOXIC if proto == "g16" else PIN_TOXIC)


def affine(proofs):
    return [{k: (G2 if k == "PiB" else G1).affine(v) for k, v in p.items()} for p in proofs]


def g16_proofs(dpk, case):
    """prove_limbs, prove_witness_limbs and a batch of 4 on one key."""
    r, s = RS[0]
    out = [dpk.prove_limbs(case.w, case.px, r, s), dpk.prove_witness_limbs(case.r1cs, case.w, r, s)]
    out += dpk.prove_witness_batch_limbs(case.r1cs, np.stack([case.w] * 4), RS)
    return out


def pin_proofs(dpk, case):
    out = [dpk.prove_limbs(case.w, case.px), dpk.prove_witness_limbs(case.r1cs, case.w)]
    out += dpk.prove_witness_batch_limbs(case.r1cs, np.stack([case.w] * 4))
    return out


def check_g16_dlogs(case, proof, r, s):
    a, b, c = case.syn.expected_dlogs(r=r, s=s)
    assert G1.affine(proof["PiA"]) == G1.affine(G1.mul_scalar(G1.G, a))
    assert G2.affine(proof["PiB"]) == G2.affine(G2.mul_scalar(G2.G, b))
    assert G1.affine(proof["PiC"]) == G1.affine(G1.mul_scalar(G1.G, c))


def check_pin_dlogs(case, proof):
    e = case.syn.expected_dlogs()
    for k in ORDER:
        assert G1.affine(proof[k]) == G1.affine(G1.mul_scalar(G1.G, e[k])), k
    assert G2.affine(proof["PiB"]) == G2.affine(G2.mul_scalar(G2.G, e["PiB"]))


def both_keys(mods, proto, case, **kw):
    """(two-step key, its Vk), (resident setup) for the same toxic values and load options."""
    groth16, snark, _ = mods
    mod = groth16 if proto == "g16" else snark
    tox = toxic_of(proto, case)
    two = mod.GenerateTrustedSetupSparse(case.r1cs, case.npublic, toxic=tox)
    load_kw = {k: kw[k] for k in ("window_bits", "rank", "world", "table_windows") if k in kw}
    old = two.load_pk(**load_kw)
    res = mod.GenerateTrustedSetupResident(case.r1cs, case.npublic, toxic=tox, **load_kw)
    return two, old, res


def assert_same_vk(proto, two, res):
    if proto == "g16":
        assert res.Vk["IC"] == two.Vk["IC"]
        assert res.Vk["G1"] == two.Vk["G1"] and res.Vk["G2"] == two.Vk["G2"]
    else:
        assert res.Vk == two.Vk


CASES = ["groth16_test", "x3x5", "chain21", "mul", "syn12", "syn16", "syn12short"]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("proto", ["g16", "pin"])
@pytest.mark.parametrize("name", CASES)
def test_resident_key_equals_the_two_step_key(mods, golden_dir, proto, name):
    groth16, snark, _ = mods
    case = make_case(mods, golden_dir, proto, name)
    two, old, res = both_keys(mods, proto, case)
    try:
        assert_same_vk(proto, two, res)
        assert res.pk.device_bytes() == old.device_bytes()
        prove = g16_proofs if proto == "g16" else pin_proofs
        got, exp = prove(res.pk, case), prove(old, case)
        assert affine(got) == affine(exp)
        assert res.pk.device_bytes() == old.device_bytes()            # the batch scratch too
        wrong = [(case.public[0] + 1) % R] + case.public[1:]
        if proto == "g16":
            assert groth16.VerifyProof(res.Vk, got[1], case.public)
            assert not groth16.VerifyProof(res.Vk, got[1], wrong)
            if case.syn is not None:
                check_g16_dlogs(case, got[1], *RS[0])
                check_g16_dlogs(case, got[5], *RS[3])
        else:
            assert snark.VerifyProof(res.Vk, got[1], case.public)
            if any(not G1.is_zero(p) for p in res.Vk["IC"][1:]):
                assert not snark.VerifyProof(res.Vk, got[1], wrong)
            else:       # IC[1..] = A[1..npublic] at infinity (a public signal outside A): no public input is bound
                assert snark.VerifyProof(res.Vk, got[1], wrong)
                assert not snark.VerifyProof(res.Vk, dict(got[1], PiH=got[1]["PiA"]), case.public)
            if case.syn is not None:
                check_pin_dlogs(case, got[1])
    finally:
        old.free()
        res.pk.free()
        case.r1cs.free()


def _config(key, value):
    from gosnark_b200._lib import check, lib
    check(lib().b200_config(key, value))


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("proto", ["g16", "pin"])
@pytest.mark.parametrize("cfg", ["acc1", "acc2", "t1", "t3", "wb9"])
def test_configurations(mods, proto, cfg):
    from gosnark_b200 import _lib
    case = synthetic_case(proto, (1 << 12) + 2)
    kw = {"t1": {"table_windows": 1}, "t3": {"table_windows": 3}, "wb9": {"window_bits": 9}}.get(cfg, {})
    if cfg.startswith("acc"):
        _config(_lib.CFG_ACC_MODE, int(cfg[3]))
    try:
        two, old, res = both_keys(mods, proto, case, **kw)
    finally:
        _config(_lib.CFG_ACC_MODE, 0)
    try:
        assert res.pk.device_bytes() == old.device_bytes()
        prove = g16_proofs if proto == "g16" else pin_proofs
        got = prove(res.pk, case)
        assert affine(got) == affine(prove(old, case))
        if proto == "g16":
            check_g16_dlogs(case, got[0], *RS[0])
        else:
            check_pin_dlogs(case, got[0])
    finally:
        old.free()
        res.pk.free()
        case.r1cs.free()


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("proto", ["g16", "pin"])
def test_context_one_key_proves_beside_a_context_zero_key(mods, proto):
    """A resident key made under B200_CFG_PK_CONTEXT = 1 proves on one host thread while a context-0 resident key proves
    on another; both proofs equal their known-discrete-log expectation."""
    from gosnark_b200 import _lib
    groth16, snark, _ = mods
    mod = groth16 if proto == "g16" else snark
    case = synthetic_case(proto, (1 << 12) + 2)
    tox = toxic_of(proto, case)
    k0 = mod.GenerateTrustedSetupResident(case.r1cs, case.npublic, toxic=tox)
    _config(_lib.CFG_PK_CONTEXT, 1)
    try:
        k1 = mod.GenerateTrustedSetupResident(case.r1cs, case.npublic, toxic=tox)
    finally:
        _config(_lib.CFG_PK_CONTEXT, 0)
    out, errs = {}, []

    def run(tag, key):
        try:
            for _ in range(4):
                out[tag] = (key.pk.prove_witness_limbs(case.r1cs, case.w, *RS[0]) if proto == "g16"
                            else key.pk.prove_witness_limbs(case.r1cs, case.w))
        except Exception as e:          # reported below
            errs.append(e)
    try:
        th = [threading.Thread(target=run, args=(t, k)) for t, k in ((0, k0), (1, k1))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errs, errs
        assert affine([out[0]]) == affine([out[1]])
        if proto == "g16":
            check_g16_dlogs(case, out[1], *RS[0])
        else:
            check_pin_dlogs(case, out[1])
    finally:
        k0.pk.free()
        k1.pk.free()
        case.r1cs.free()


def _shard_info(handle):
    from gosnark_b200._lib import check, lib, ptr
    out = np.zeros(12, dtype=np.uint64)
    check(lib().b200_groth16_shard_info(handle, ptr(out)))
    return [int(x) for x in out]


def _g16_records(keys, case, r, s):
    """Every rank's 1 KB partial record (b200_groth16_prove_witness_device without a communicator) and their finalize."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, lib, ptr
    L = lib()
    rr, ss = ints_to_limbs([r]), ints_to_limbs([s])
    d_w = torch.from_numpy(case.w.reshape(-1).view(np.int64)).cuda()
    parts = torch.zeros(128 * len(keys), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for g, h in enumerate(keys):
        check(L.b200_groth16_prove_witness_device(h, case.r1cs.handle, d_w.data_ptr(), case.m, ptr(rr), ptr(ss),
                                                  parts[128 * g:].data_ptr(), None))
    d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
    check(L.b200_groth16_finalize_device(keys[0], parts.data_ptr(), len(keys), ptr(rr), ptr(ss), d_out.data_ptr(), None))
    torch.cuda.synchronize()
    return parts.cpu().numpy().view(np.uint64).copy(), d_out.cpu().numpy().view(np.uint64).copy()


def _pin_records(keys, case):
    import torch
    from gosnark_b200._lib import check, lib
    L = lib()
    d_w = torch.from_numpy(case.w.reshape(-1).view(np.int64)).cuda()
    recs = torch.zeros(256 * len(keys), dtype=torch.int64, device="cuda")
    d_out = torch.zeros(108, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for g, h in enumerate(keys):
        check(L.b200_pinocchio_prove_witness_batch_record_device(h, case.r1cs.handle, d_w.data_ptr(), case.m, 1,
                                                                 recs[256 * g:].data_ptr(), None))
    check(L.b200_pinocchio_finalize_records_batch_device(recs.data_ptr(), len(keys), 1, d_out.data_ptr(), None))
    torch.cuda.synchronize()
    return recs.cpu().numpy().view(np.uint64).copy(), d_out.cpu().numpy().view(np.uint64).copy()


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("proto", ["g16", "pin"])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_shards(mods, proto, world):
    """Each rank of a shard emulated on one GPU: its resident key has the two-step key's shard info and device bytes; the
    ranks' records finalize to the two-step shards' proof and to the unsharded proof."""
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    groth16, snark, _ = mods
    mod = groth16 if proto == "g16" else snark
    case = synthetic_case(proto, (1 << 12) + 2)
    tox = toxic_of(proto, case)
    two = mod.GenerateTrustedSetupSparse(case.r1cs, case.npublic, toxic=tox)
    olds = [two.load_pk(rank=g, world=world) for g in range(world)]
    news = [mod.GenerateTrustedSetupResident(case.r1cs, case.npublic, toxic=tox, rank=g, world=world).pk for g in range(world)]
    whole = mod.GenerateTrustedSetupResident(case.r1cs, case.npublic, toxic=tox).pk
    try:
        for a, b in zip(olds, news):
            assert a.device_bytes() == b.device_bytes()
            if proto == "g16":
                assert _shard_info(a.handle) == _shard_info(b.handle)
        if proto == "g16":
            r, s = RS[0]
            split = lambda w: dict(zip(("PiA", "PiC"), _unflatten_g1(w[:24])), PiB=_unflatten_g2(w[24:48])[0])
            out_new = split(_g16_records([k.handle for k in news], case, r, s)[1])
            out_old = split(_g16_records([k.handle for k in olds], case, r, s)[1])
            assert affine([out_new]) == affine([out_old])
            pa, pb, pc = out_new["PiA"], out_new["PiB"], out_new["PiC"]
            ref = whole.prove_witness_limbs(case.r1cs, case.w, r, s)
            assert (G1.affine(pa), G2.affine(pb), G1.affine(pc)) == (G1.affine(ref["PiA"]), G2.affine(ref["PiB"]),
                                                                     G1.affine(ref["PiC"]))
            check_g16_dlogs(case, {"PiA": pa, "PiB": pb, "PiC": pc}, r, s)
        else:
            split = lambda w: dict(zip(ORDER, _unflatten_g1(w[:84])), PiB=_unflatten_g2(w[84:108])[0])
            proof = split(_pin_records([k.handle for k in news], case)[1])
            assert affine([proof]) == affine([split(_pin_records([k.handle for k in olds], case)[1])])
            ref = whole.prove_witness_limbs(case.r1cs, case.w)
            assert all(G1.affine(proof[k]) == G1.affine(ref[k]) for k in ORDER)
            check_pin_dlogs(case, proof)
    finally:
        for k in olds + news + [whole]:
            k.free()
        case.r1cs.free()


SCALE_SCRIPT = r"""
import json, sys, threading, time
sys.path.insert(0, {root!r})
from gosnark_b200 import _lib, groth16, snark
from gosnark_b200.synthetic import CircuitGroth16, CircuitPinocchio
from oracle import ref_py as o
proto, mode = sys.argv[1], sys.argv[2]
_lib.init()
n = 1 << 20
syn = CircuitGroth16(n=n, mint=False) if proto == "g16" else CircuitPinocchio(n, mint=False)
mod = groth16 if proto == "g16" else snark

def rss():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) * 1024
peak, stop = [0], [False]
def sample():
    while not stop[0]:
        peak[0] = max(peak[0], rss())
        time.sleep(0.002)
base = rss()
th = threading.Thread(target=sample)
th.start()
if mode == "resident":
    pk = mod.GenerateTrustedSetupResident(syn.r1cs, syn.npublic, toxic=syn.toxic).pk
else:
    pk = mod.GenerateTrustedSetupSparse(syn.r1cs, syn.npublic, toxic=syn.toxic).load_pk()
peak[0] = max(peak[0], rss())
stop[0] = True
th.join()
ok = True
if mode == "resident":
    G1, G2 = o.BN.G1, o.BN.G2
    if proto == "g16":
        r, s = syn.r, syn.s
        p = pk.prove_witness_limbs(syn.r1cs, syn.w, r, s)
        a, b, c = syn.expected_dlogs(r=r, s=s)
        ok = (G1.affine(p["PiA"]) == G1.affine(G1.mul_scalar(G1.G, a)) and
              G2.affine(p["PiB"]) == G2.affine(G2.mul_scalar(G2.G, b)) and
              G1.affine(p["PiC"]) == G1.affine(G1.mul_scalar(G1.G, c)))
    else:
        p = pk.prove_witness_limbs(syn.r1cs, syn.w)
        e = syn.expected_dlogs()
        ok = all(G1.affine(p[k]) == G1.affine(G1.mul_scalar(G1.G, e[k])) for k in {order!r})
        ok = ok and G2.affine(p["PiB"]) == G2.affine(G2.mul_scalar(G2.G, e["PiB"]))
pk.free()
print(json.dumps({{"growth": peak[0] - base, "ok": ok}}))
"""


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("proto", ["g16", "pin"])
def test_scale_2p20_host_memory(proto):
    """At 2^20 (Groth16 with full tables, and Pinocchio), in a subprocess each: the resident key's proof equals its
    known-discrete-log expectation, and the call's peak VmRSS growth is under a tenth of the two-step path's growth,
    which is at least 0.6 GB (the host CRS)."""
    script = SCALE_SCRIPT.format(root=ROOT, order=ORDER)
    res = {}
    for mode in ("twostep", "resident"):
        p = subprocess.run([sys.executable, "-c", script, proto, mode], capture_output=True, text=True, cwd=ROOT, timeout=1700)
        assert p.returncode == 0, p.stderr[-3000:]
        res[mode] = json.loads(p.stdout.strip().splitlines()[-1])
    assert res["resident"]["ok"]
    assert res["twostep"]["growth"] >= 0.6e9, res
    assert res["resident"]["growth"] < res["twostep"]["growth"] / 10, res


def test_errors(mods):
    """Every error of the header's contract, each followed by a valid call that succeeds; a failed call leaves no
    handle."""
    import ctypes
    from gosnark_b200._lib import _h, ints_to_limbs, lib, ptr
    groth16, snark, r1csqap = mods
    n, m = len(A), len(A[0])
    sp = r1csqap.SparseR1CS(n, m, (A, B, C))
    rp = np.array([0, 1, 2], dtype=np.uint32)
    tiny = r1csqap.SparseR1CS(2, 2, [(rp, np.array([0, 1], dtype=np.uint32), [1, 1])] * 3)      # m = 2 < 3
    L = lib()
    bufs = [np.zeros((64, 24), dtype=np.uint64) for _ in range(6)]
    G16N = ("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta")
    PINN = ("T", "Ka", "Kb", "Kc", "Kbeta", "Kgamma", "RhoA", "RhoB")

    def call(proto, hnd, npub, tox, wb=0, rank=0, world=1, null=None, null_toxic=False, null_out=False):
        names = G16N if proto == "g16" else PINN
        outs = [ptr(b) for b in bufs[:5 if proto == "g16" else 3]]
        if null is not None:
            outs[null] = None
        h = _h(0)
        tl = None if null_toxic else ptr(ints_to_limbs([tox[k] for k in names]))
        fn = L.b200_groth16_setup_pk if proto == "g16" else L.b200_pinocchio_setup_pk
        rc = fn(hnd, npub, tl, wb, rank, world, None if null_out else ctypes.byref(h), *outs)
        return rc, h.value

    def valid(proto):
        tox = G16_TOXIC if proto == "g16" else PIN_TOXIC
        rc, h = call(proto, sp.handle, 1, tox)
        assert rc == 0 and h
        assert L.b200_pk_free(h) == 0

    try:
        for proto, tox, nout in (("g16", G16_TOXIC, 5), ("pin", PIN_TOXIC, 3)):
            names = G16N if proto == "g16" else PINN
            cases = [((sp.handle + 1000, 1, tox), {}, EINVAL), ((tiny.handle, 0, tox), {}, EINVAL),
                     ((sp.handle, m, tox), {}, EINVAL), ((sp.handle, m + 5, tox), {}, EINVAL),
                     ((sp.handle, 1, tox), {"null_toxic": True}, EINVAL), ((sp.handle, 1, tox), {"null_out": True}, EINVAL)]
            cases += [((sp.handle, 1, tox), {"null": k}, EINVAL) for k in range(nout)]
            for k in names:                                                   # a toxic value >= r
                cases.append(((sp.handle, 1, dict(tox, **{k: R})), {}, ERANGE))
            for t in (1, n):                                                  # T is an interpolation point
                cases.append(((sp.handle, 1, dict(tox, T=t)), {}, EINVAL))
            if proto == "g16":
                cases += [((sp.handle, 1, dict(tox, Kgamma=0)), {}, EINVAL), ((sp.handle, 1, dict(tox, Kdelta=0)), {}, EINVAL)]
            cases += [((sp.handle, 1, tox), {"rank": -1, "world": 2}, EINVAL), ((sp.handle, 1, tox), {"rank": 2, "world": 2}, EINVAL),
                      ((sp.handle, 1, tox), {"rank": 0, "world": 0}, EINVAL), ((sp.handle, 1, tox), {"wb": 1}, EINVAL),
                      ((sp.handle, 1, tox), {"wb": 25}, EINVAL)]
            for args, kw, code in cases:
                rc, h = call(proto, *args, **kw)
                assert (rc, h) == (code, 0), (proto, args[1:], kw, rc, h)
                valid(proto)
        with pytest.raises(ValueError):
            groth16.GenerateTrustedSetupResident(sp, 1, world=2)
        with pytest.raises(ValueError):
            snark.GenerateTrustedSetupResident(sp, 1, world=2)
    finally:
        sp.free()
        tiny.free()
