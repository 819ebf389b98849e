"""GPU: the trusted setup from a sparse R1CS (b200_groth16_setup, b200_pinocchio_setup; groth16 / snark
GenerateTrustedSetupSparse).

Small circuits are compared with the dense GenerateTrustedSetup, which is itself X,Y,Z-exact with the oracle; larger ones
with CircuitGroth16 / CircuitPinocchio, whose discrete logs are Python ints and whose points come from the
reference-order kernel.  Points are compared as group elements (affine coordinates)."""
import json
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = o.R
G1, G2 = o.BN.G1, o.BN.G2
EINVAL, ERANGE = -3, -4

# groth16_test.go:20-28 circuit (y = x^3 + x + 5): n = 7 constraints, m = 8 signals
A = [[0, 0, 1, 0, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0, 0, 0], [0, 0, 1, 0, 1, 0, 0, 0], [5, 0, 0, 0, 0, 1, 0, 0],
     [0, 0, 0, 0, 0, 0, 1, 0], [0, 1, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0]]
B = [[0, 0, 1, 0, 0, 0, 0, 0], [0, 0, 1, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0],
     [1, 0, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0]]
C = [[0, 0, 0, 1, 0, 0, 0, 0], [0, 0, 0, 0, 1, 0, 0, 0], [0, 0, 0, 0, 0, 1, 0, 0], [0, 0, 0, 0, 0, 0, 1, 0],
     [0, 1, 0, 0, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0, 1, 0], [0, 0, 0, 0, 0, 0, 0, 1]]
W = [1, 35, 3, 9, 27, 30, 35, 1]
G16_TOXIC = {"T": 0x1234567890abcdef1234567890abcdef, "Kalpha": 0x1111, "Kbeta": 0x2222222222, "Kgamma": 0x3333,
             "Kdelta": 0x444444}
PIN_TOXIC = {"T": 0x7777777777abcdef12, "Ka": 0x11, "Kb": 0x2222, "Kc": 0x333333, "Kbeta": 0x44, "Kgamma": 0x5555,
             "RhoA": 0x666666, "RhoB": 0x77}


@pytest.fixture(scope="module")
def mods():
    from gosnark_b200 import _lib, groth16, r1csqap, snark
    _lib.init()
    return groth16, snark, r1csqap


def aff(G, p):
    """A point as a group element: affine (x, y), or None for infinity."""
    return None if G.is_zero(p) else tuple(G.affine(p)[:2])


def aff_list(G, pts):
    return [aff(G, p) for p in pts]


def small_circuits(golden_dir):
    out = [("groth16_test", A, B, C, 1)]
    for name in ("x3x5", "chain21", "mul"):
        with open(os.path.join(golden_dir, f"gobin_{name}.json")) as f:
            cc = json.load(f)["compiledcircuit"]
        out.append((name, cc["R1CS"]["A"], cc["R1CS"]["B"], cc["R1CS"]["C"], cc["NPublic"]))
    return out


@pytest.mark.parametrize("k", range(4), ids=["groth16_test", "x3x5", "chain21", "mul"])
def test_small_circuits_equal_the_dense_setup(mods, golden_dir, k):
    """Every array of both sparse setups equals the dense GenerateTrustedSetup's as group elements, and Z is equal.  The
    golden circuits x3x5 and chain21 have m = n + 1, so Z (m - 2 roots) differs from the domain polynomial (n roots)."""
    groth16, snark, r1csqap = mods
    name, a, b, c, npub = small_circuits(golden_dir)[k]
    n, m = len(a), len(a[0])
    pf = r1csqap.PolynomialField()
    alphas, betas, gammas, _ = pf.R1CSToQAP(a, b, c)
    circuit = {"NVars": m, "NPublic": npub}
    sp = r1csqap.SparseR1CS(n, m, (a, b, c))
    try:
        dense = groth16.GenerateTrustedSetup(m, circuit, alphas, betas, gammas, toxic=G16_TOXIC)
        new = groth16.GenerateTrustedSetupSparse(sp, npub, toxic=G16_TOXIC)
        dpk, npk = dense["Pk"], new.pk_dict()
        assert npk["Z"] == dpk["Z"] and len(npk["Z"]) == m - 1
        for key in ("BACDelta", "PowersTauDelta"):
            assert aff_list(G1, npk[key]) == aff_list(G1, dpk[key]), key
        for key in ("Alpha", "Beta", "Delta"):
            assert aff(G1, npk["G1"][key]) == aff(G1, dpk["G1"][key]), key
        for key in ("At", "BACGamma"):
            assert aff_list(G1, npk["G1"][key]) == aff_list(G1, dpk["G1"][key]), key
        assert aff_list(G2, npk["G2"]["BACGamma"]) == aff_list(G2, dpk["G2"]["BACGamma"])
        for key in ("Beta", "Delta"):
            assert aff(G2, npk["G2"][key]) == aff(G2, dpk["G2"][key]), key
        assert aff_list(G1, new.Vk["IC"]) == aff_list(G1, dense["Vk"]["IC"])
        for key in ("Beta", "Gamma", "Delta"):
            assert aff(G2, new.Vk["G2"][key]) == aff(G2, dense["Vk"]["G2"][key]), key
        assert aff(G1, new.Vk["G1"]["Alpha"]) == aff(G1, dense["Vk"]["G1"]["Alpha"])
        assert all(p[2] == 1 for p in npk["G1"]["At"] if not G1.is_zero(p))      # affine (x, y, 1)
        if name == "groth16_test":                       # pk_dict() is a key GenerateProofs takes; the Vk verifies it
            px = pf.CombinePolynomials(W, alphas, betas, gammas)[3]
            proof = groth16.GenerateProofs(circuit, npk, W, px)
            assert groth16.VerifyProof(new.Vk, proof, [35]) and not groth16.VerifyProof(new.Vk, proof, [34])
            groth16.Forget(npk)

        dense = snark.GenerateTrustedSetup(m, circuit, alphas, betas, gammas, toxic=PIN_TOXIC)
        new = snark.GenerateTrustedSetupSparse(sp, npub, toxic=PIN_TOXIC)
        dpk, npk = dense["Pk"], new.pk_dict()
        assert npk["Z"] == dpk["Z"]
        for key in ("A", "Ap", "Bp", "C", "Cp", "Kp", "G1T"):
            assert aff_list(G1, npk[key]) == aff_list(G1, dpk[key]), key
        assert aff_list(G2, npk["B"]) == aff_list(G2, dpk["B"])
        for key in ("Vkb", "G1Kbg"):
            assert aff(G1, new.Vk[key]) == aff(G1, dense["Vk"][key]), key
        for key in ("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz"):
            assert aff(G2, new.Vk[key]) == aff(G2, dense["Vk"][key]), key
        assert aff_list(G1, new.Vk["IC"]) == aff_list(G1, dense["Vk"]["IC"])
        assert new.Toxic["RhoC"] == dense["Toxic"]["RhoC"]
    finally:
        sp.free()


def gpu_affine(group, jac):
    """(k, 12|24) Jacobian limbs -> (k, 8|16) affine limbs by the reference-formula kernel, infinity (0, 0)."""
    from gosnark_b200._lib import check, lib, ptr
    jac = np.ascontiguousarray(jac, dtype=np.uint64)
    w = 8 if group == 1 else 16
    out = np.zeros((jac.shape[0], w), dtype=np.uint64)
    fn = lib().b200_g1_affine_batch if group == 1 else lib().b200_g2_affine_batch
    check(fn(ptr(jac), jac.shape[0], ptr(out)))
    return out


def assert_same_points(group, new, ref, what):
    """new: affine (x, y, 1) limbs from the sparse setup; ref: Jacobian limbs of the same group elements."""
    w = 8 if group == 1 else 16
    new = np.asarray(new, dtype=np.uint64).reshape(-1, 3 * w // 2)
    ref = np.asarray(ref, dtype=np.uint64).reshape(-1, 3 * w // 2)
    assert new.shape == ref.shape, what
    exp = gpu_affine(group, ref)
    assert np.array_equal(new[:, :w], exp), what
    inf = ~exp.any(axis=1)
    one = np.zeros(w // 2, dtype=np.uint64)
    one[0] = 1
    assert (new[inf, w:] == 0).all() and (new[~inf, w:] == one).all(), what


_groth = {}


def circuit_groth16(n):
    from gosnark_b200.synthetic import CircuitGroth16
    if n not in _groth:
        _groth[n] = CircuitGroth16(n=n)
    return _groth[n]


def go_groth16_verify(vk, proof, public):
    binary = os.path.join(ROOT, "oracle", "_ref", "go-snark-cli")
    if not os.path.exists(binary):
        return None
    g2 = lambda p: [list(c) for c in p]
    vk_json = {"IC": [list(p) for p in vk["IC"]], "G1": {"Alpha": list(vk["G1"]["Alpha"])},
               "G2": {k: g2(vk["G2"][k]) for k in ("Beta", "Gamma", "Delta")}}
    proof_json = {"PiA": list(proof["PiA"]), "PiB": g2(proof["PiB"]), "PiC": list(proof["PiC"])}
    d = tempfile.mkdtemp(prefix="gss_")
    try:
        b = os.path.join(d, "gsc")
        shutil.copy(binary, b)
        os.chmod(b, 0o755)
        for fname, obj in (("trustedsetup.json", {"Vk": vk_json}), ("publicInputs.json", public), ("proofs.json", proof_json),
                           ("compiledcircuit.json", {})):
            with open(os.path.join(d, fname), "w") as f:
                json.dump(obj, f)
        p = subprocess.run([b, "groth16", "verify"], cwd=d, capture_output=True, text=True, timeout=300)
        return p.stdout + p.stderr
    finally:
        shutil.rmtree(d)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("n", [(1 << 12) + 2, 1 << 16], ids=["4098", "65536"])
def test_groth16_at_scale(mods, n):
    """Every point equals CircuitGroth16's; proofs from b200_groth16_prove and b200_groth16_prove_witness on the new key
    verify under the new Vk, a wrong public input is rejected, and (n = 2^12 + 2) go-snark-cli accepts the proof."""
    groth16 = mods[0]
    syn = circuit_groth16(n)
    new = groth16.GenerateTrustedSetupSparse(syn.r1cs, syn.npublic, toxic=syn.toxic)
    for key, ref in (("at", syn.at), ("b1", syn.b1), ("bacdelta", syn.cd), ("ptd", syn.ptd), ("ic", syn.ic),
                     ("alpha1", syn.alpha1), ("beta1", syn.beta1), ("delta1", syn.delta1)):
        assert_same_points(1, getattr(new, key), ref, key)
    for key, ref in (("b2", syn.b2), ("beta2", syn.beta2), ("gamma2", syn.gamma2), ("delta2", syn.delta2)):
        assert_same_points(2, getattr(new, key), ref, key)
    assert np.array_equal(new.z, syn.z[: syn.m - 1])
    dpk = new.load_pk()
    try:
        pub = syn.circuit.public_signals
        p_px = dpk.prove_limbs(syn.w, syn.px, syn.r, syn.s)
        p_w = dpk.prove_witness_limbs(syn.r1cs, syn.w, syn.r, syn.s)
        exp = [G.affine(G.mul_scalar(G.G, d)) for G, d in zip((G1, G2, G1), syn.expected_dlogs())]
        for p in (p_px, p_w):
            assert [G1.affine(p["PiA"]), G2.affine(p["PiB"]), G1.affine(p["PiC"])] == exp
            assert groth16.VerifyProof(new.Vk, p, pub)
        assert not groth16.VerifyProof(new.Vk, p_w, [(pub[0] + 1) % R])
        if n == (1 << 12) + 2:
            out = go_groth16_verify(new.Vk, p_w, pub)
            if out is not None:
                assert "Proofs verified" in out and "not verified" not in out, out
    finally:
        dpk.free()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("n", [(1 << 12) + 2, 1 << 16], ids=["4098", "65536"])
def test_pinocchio_at_scale(mods, n):
    """Every point equals CircuitPinocchio's, and a proof on the new key verifies under the new Vk (snark.VerifyProof)."""
    from gosnark_b200.synthetic import CircuitPinocchio
    snark = mods[1]
    syn = CircuitPinocchio(n)
    try:
        new = snark.GenerateTrustedSetupSparse(syn.r1cs, syn.npublic, toxic=syn.toxic)
        for key in ("A", "Ap", "Bp", "C", "Cp", "Kp", "G1T"):
            assert_same_points(1, getattr(new, key.lower()), syn.pk[key], key)
        assert_same_points(2, new.b2, syn.pk["B"], "B")
        from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
        assert_same_points(1, new.vk_g1, _flatten_g1([syn.vk[k] for k in ("Vkb", "G1Kbg")]), "vk_g1")
        assert_same_points(2, new.vk_g2, _flatten_g2([syn.vk[k] for k in ("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz")]), "vk_g2")
        assert np.array_equal(new.z, syn.z[: syn.m - 1])
        dpk = new.load_pk()
        try:
            proof = dpk.prove_limbs(syn.w, syn.px)
            assert snark.VerifyProof(new.Vk, proof, syn.circuit.public_signals)
        finally:
            dpk.free()
    finally:
        syn.r1cs.free()


def test_sharded_key_gives_the_unsharded_proof(mods):
    """The new Groth16 key loaded as 2 shards (b200_groth16_pk_load_shard) and its records summed by
    b200_groth16_finalize_device give the unsharded key's proof."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, lib, ptr
    groth16 = mods[0]
    syn = circuit_groth16((1 << 12) + 2)
    new = groth16.GenerateTrustedSetupSparse(syn.r1cs, syn.npublic, toxic=syn.toxic)
    single = new.load_pk()
    shards = [new.load_pk(rank=rk, world=2) for rk in range(2)]
    L = lib()
    rr, ss = ints_to_limbs([syn.r]), ints_to_limbs([syn.s])
    try:
        d_w = torch.from_numpy(syn.w.reshape(-1).view(np.int64)).cuda()
        torch.cuda.synchronize()
        parts = torch.zeros(256, dtype=torch.int64, device="cuda")
        for rk, pk in enumerate(shards):
            check(L.b200_groth16_prove_witness_device(pk.handle, syn.r1cs.handle, d_w.data_ptr(), syn.m, ptr(rr), ptr(ss),
                                                      parts[128 * rk:].data_ptr(), None))
        d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
        check(L.b200_groth16_finalize_device(shards[0].handle, parts.data_ptr(), 2, ptr(rr), ptr(ss), d_out.data_ptr(), None))
        torch.cuda.synchronize()
        from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
        words = d_out.cpu().numpy().view(np.uint64)
        pa, pc = _unflatten_g1(words[:24])
        pb = _unflatten_g2(words[24:48])[0]
        ref = single.prove_witness_limbs(syn.r1cs, syn.w, syn.r, syn.s)
        assert (G1.affine(pa), G2.affine(pb), G1.affine(pc)) == (G1.affine(ref["PiA"]), G2.affine(ref["PiB"]),
                                                                 G1.affine(ref["PiC"]))
    finally:
        for pk in [single] + shards:
            pk.free()


def test_argument_errors(mods):
    """Every B200_EINVAL / B200_ERANGE case of the header, each followed by a valid setup that succeeds."""
    from gosnark_b200._lib import B200Error, ints_to_limbs, lib, ptr
    groth16, snark, r1csqap = mods
    n, m = len(A), len(A[0])
    sp = r1csqap.SparseR1CS(n, m, (A, B, C))
    rp = np.array([0, 1, 2], dtype=np.uint32)
    tiny = r1csqap.SparseR1CS(2, 2, [(rp, np.array([0, 1], dtype=np.uint32), [1, 1])] * 3)      # m = 2 < 3
    L = lib()
    bufs = [np.zeros((64, 24), dtype=np.uint64) for _ in range(16)]

    def g16(h, npub, tox, null=None):
        names = ("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta")
        args = [ptr(b) for b in bufs[:13]]
        if null is not None:
            args[null] = None
        return L.b200_groth16_setup(h, npub, ptr(ints_to_limbs([tox[k] for k in names])), *args)

    def pin(h, npub, tox, null=None):
        names = ("T", "Ka", "Kb", "Kc", "Kbeta", "Kgamma", "RhoA", "RhoB")
        args = [ptr(b) for b in bufs[:11]]
        if null is not None:
            args[null] = None
        return L.b200_pinocchio_setup(h, npub, ptr(ints_to_limbs([tox[k] for k in names])), *args)

    def valid():
        assert groth16.GenerateTrustedSetupSparse(sp, 1, toxic=G16_TOXIC).at.shape == (m, 12)
        assert snark.GenerateTrustedSetupSparse(sp, 1, toxic=PIN_TOXIC).a.shape == (m, 12)

    try:
        cases = []
        for fn, tox, nout in ((g16, G16_TOXIC, 13), (pin, PIN_TOXIC, 11)):
            cases += [(fn, (sp.handle + 1000, 1, tox), EINVAL), (fn, (tiny.handle, 0, tox), EINVAL),
                      (fn, (sp.handle, m, tox), EINVAL), (fn, (sp.handle, m + 5, tox), EINVAL)]
            cases += [(fn, (sp.handle, 1, tox, k), EINVAL) for k in range(nout)]
            for key in tox:
                cases.append((fn, (sp.handle, 1, dict(tox, **{key: R})), ERANGE))
                cases.append((fn, (sp.handle, 1, dict(tox, **{key: (1 << 256) - 1})), ERANGE))
            for t in (1, 2, n):                                              # T in {1..n}
                cases.append((fn, (sp.handle, 1, dict(tox, T=t)), EINVAL))
        cases += [(g16, (sp.handle, 1, dict(G16_TOXIC, Kgamma=0)), EINVAL), (g16, (sp.handle, 1, dict(G16_TOXIC, Kdelta=0)), EINVAL)]
        for fn, args, code in cases:
            assert fn(*args) == code, (fn.__name__, args[:2], code)
            valid()
        assert L.b200_groth16_setup(sp.handle, 1, None, *[ptr(b) for b in bufs[:13]]) == EINVAL
        assert L.b200_pinocchio_setup(sp.handle, 1, None, *[ptr(b) for b in bufs[:11]]) == EINVAL
        valid()
        # T = n + 1 and T = 0 lie outside the domain: valid; through Python a bad value raises B200Error
        assert g16(sp.handle, 1, dict(G16_TOXIC, T=n + 1)) == 0 and g16(sp.handle, 1, dict(G16_TOXIC, T=0)) == 0
        with pytest.raises(B200Error):
            groth16.GenerateTrustedSetupSparse(sp, 1, toxic=dict(G16_TOXIC, Kdelta=R + 1))
        tox = groth16.GenerateTrustedSetupSparse(sp, 1).Toxic
        assert not 1 <= tox["T"] <= n and all(0 <= v < R for v in tox.values())
    finally:
        sp.free()
        tiny.free()
