"""GPU: the verifier side (SURVEY §8f row 2) — bn128.Pairing and groth16.VerifyProof on the device, bit-exact
against the snarkjs golden (K8), the reference's own test literals (bn128/bn128_test.go:45-67) and the oracle."""
import json
import os
import random

import pytest

from oracle import ref_py as o
from test_gpu_setup_flow import A, B, C, W

pytestmark = pytest.mark.gpu
R = o.R
G1, G2 = o.BN.G1, o.BN.G2


@pytest.fixture(scope="module")
def mods():
    from gosnark_b200 import _lib, bn128, groth16, r1csqap
    _lib.init()
    return bn128.Bn128(), groth16, r1csqap.PolynomialField()


def _circom(golden_dir):
    c = json.load(open(os.path.join(golden_dir, "circom_groth16.json")))
    vk, pr = c["vk"], c["proof"]
    i3 = lambda p: tuple(int(x) for x in p)
    i32 = lambda p: tuple(tuple(int(x) for x in q) for q in p)
    ovk = {"IC": [i3(p) for p in vk["IC"]], "G1": {"Alpha": i3(vk["vk_alfa_1"])},
           "G2": {"Beta": i32(vk["vk_beta_2"]), "Gamma": i32(vk["vk_gamma_2"]), "Delta": i32(vk["vk_delta_2"])}}
    proof = {"PiA": i3(pr["pi_a"]), "PiB": i32(pr["pi_b"]), "PiC": i3(pr["pi_c"])}
    gold = tuple(tuple(tuple(int(x) for x in f2) for f2 in f6) for f6 in vk["vk_alfabeta_12"])
    return ovk, proof, [int(x) for x in c["public"]], gold


def test_k8_golden_pairing(mods, golden_dir):
    """e(vk_alfa_1, vk_beta_2) == vk_alfabeta_12 (externalVerif/circom-test/verification_key.json:62-91)."""
    bn, _, _ = mods
    vk, _, _, gold = _circom(golden_dir)
    assert bn.Pairing(vk["G1"]["Alpha"], vk["G2"]["Beta"]) == gold


def test_reference_pairing_literal_and_bilinearity(mods):
    """bn128_test.go:45-67: e(25 G1, 30 G2) == e(30 G1, 25 G2), with the first coefficient the test prints."""
    bn, _, _ = mods
    p1, q1 = G1.mul_scalar(G1.G, 25), G2.mul_scalar(G2.G, 30)      # Jacobian, Z != 1: the kernel normalises like preComputeG1
    p2, q2 = G1.mul_scalar(G1.G, 30), G2.mul_scalar(G2.G, 25)
    e1, e2 = bn.PairingBatch([p1, p2], [q1, q2])
    assert e1 == e2 == o.BN.pairing(p1, q1)
    assert e1[0][0][0] == 8016119724813186033542830391460394070015218389456422587891475873290878009957


def test_pairing_batch_vs_oracle_and_infinity(mods):
    bn, _, _ = mods
    rng = random.Random(5)
    ps = [G1.mul_scalar(G1.G, rng.randrange(1, R)) for _ in range(2)] + [G1.zero3()]
    qs = [G2.mul_scalar(G2.G, rng.randrange(1, R)) for _ in range(2)] + [G2.G]
    got = bn.PairingBatch(ps, qs)
    for p, q, e in zip(ps, qs, got):
        assert e == o.BN.pairing(p, q)
    assert bn.PairingBatch([], []) == []
    with pytest.raises(Exception, match="Fq2.One"):           # the reference panics (bn128.go:238-241)
        bn.Pairing(G1.G, G2.zero3())
    with pytest.raises(Exception, match=">= q"):
        bn.Pairing((o.Q, 2, 1), G2.G)


def test_verify_circom_proof(mods, golden_dir):
    """externalVerif/circomVerifier_test.go:9-13: the snarkjs proof verifies; a wrong public input does not."""
    _, groth16, _ = mods
    vk, proof, public, _ = _circom(golden_dir)
    assert groth16.VerifyProof(vk, proof, public, True)
    assert not groth16.VerifyProof(vk, proof, [public[0] + 1], True)
    bad = dict(proof, PiC=G1.double(proof["PiC"]))
    assert not groth16.VerifyProof(vk, bad, public)


def test_minimal_flow_all_gpu(mods):
    """TestGroth16MinimalFlow (groth16/groth16_test.go:16-107) with every step on the GPU, verify included."""
    _, groth16, pf = mods
    circuit = {"NVars": 8, "NPublic": 1}
    alphas, betas, gammas, _ = pf.R1CSToQAP(A, B, C)
    _, _, _, px = pf.CombinePolynomials(W, alphas, betas, gammas)
    setup = groth16.GenerateTrustedSetup(len(W), circuit, alphas, betas, gammas)
    proof = groth16.GenerateProofs(circuit, setup["Pk"], W, px)
    assert groth16.VerifyProof(setup["Vk"], proof, [35])                 # :100
    assert not groth16.VerifyProof(setup["Vk"], proof, [34])             # :106
    assert o.groth16_verify(setup["Vk"], proof, [35])
    with pytest.raises(Exception):
        groth16.VerifyProof(setup["Vk"], proof, [35, 1, 2])              # more signals than IC entries


def test_verify_many_public_signals_edge_values(mods):
    """icPubl = IC[0] + sum publicSignals[i]*IC[i+1] (groth16.go:283-286) with eight signals — 0, 1, r-1, 2^128-ish values on
    either side of the GLV split, random full-width ones — on a verification key and proof built from known discrete logs
    so that e(A,B) == e(alpha,beta) * e(icPubl,gamma) * e(C,delta) holds exactly: accepted (device and oracle), rejected
    when any one signal moves, and an odd signal count exercises the half-empty warp of k_ic_terms."""
    _, groth16, _ = mods
    rng = random.Random(77)
    rnd = lambda: rng.randrange(1, R)
    for pubs in ([0, 1, R - 1, (1 << 128) - 1, 1 << 128, rnd(), rnd(), rnd()], [rnd(), 0, rnd()], [R - 2]):
        al, be, ga, de, a, b = (rnd() for _ in range(6))
        ic = [rnd() for _ in range(len(pubs) + 1)]
        ic_pub = (ic[0] + sum(p * k for p, k in zip(pubs, ic[1:]))) % R
        c = (a * b - al * be - ic_pub * ga) * pow(de, -1, R) % R
        g1 = lambda k: G1.mul_scalar(G1.G, k)
        g2 = lambda k: G2.mul_scalar(G2.G, k)
        vk = {"IC": [g1(k) for k in ic], "G1": {"Alpha": g1(al)}, "G2": {"Beta": g2(be), "Gamma": g2(ga), "Delta": g2(de)}}
        proof = {"PiA": g1(a), "PiB": g2(b), "PiC": g1(c)}
        assert groth16.VerifyProof(vk, proof, pubs)
        for j in range(len(pubs)):
            moved = list(pubs)
            moved[j] = (moved[j] + 1) % R
            assert not groth16.VerifyProof(vk, proof, moved), j
        assert groth16.VerifyProof(vk, proof, [p + R for p in pubs])          # p + r: MulScalar's walk gives p for these p (not for all)
    assert o.groth16_verify(vk, proof, pubs)


def test_fq12_mul_batch(mods):
    """fields/fq12.go:72-84 on the device, against the oracle (random elements and the identity)."""
    bn, _, _ = mods
    rng = random.Random(12)
    rnd = lambda: tuple(tuple((rng.randrange(o.Q), rng.randrange(o.Q)) for _ in range(3)) for _ in range(2))
    one = (((1, 0), (0, 0), (0, 0)), ((0, 0), (0, 0), (0, 0)))
    xs, ys = [rnd(), rnd(), one], [rnd(), one, rnd()]
    got = bn.Fq12MulBatch(xs, ys)
    assert got == [o.BN.Fq12.mul(x, y) for x, y in zip(xs, ys)]
    assert got[1] == xs[1] and got[2] == ys[2]


def test_pinocchio_setup_and_verify_on_gpu(mods, golden_dir):
    """snark.GenerateTrustedSetup (snark.go:98-251) minted on the GPU equals the oracle X,Y,Z-exactly for injected toxic
    values; the GPU proof under it passes snark.VerifyProof (:292-372) on the GPU and the oracle's; the Go binary's own
    Pinocchio proof verifies too, and a wrong public input fails at the QAP check like the reference."""
    from gosnark_b200 import snark
    g = json.load(open(os.path.join(golden_dir, "gobin_x3x5.json")))
    cc = g["compiledcircuit"]
    r1 = cc["R1CS"]
    _, _, pf = mods
    alphas, betas, gammas, _ = pf.R1CSToQAP(r1["A"], r1["B"], r1["C"])
    tox = {"T": 0x1234567, "Ka": 0x1111, "Kb": 0x2222, "Kc": 0x3333, "Kbeta": 0x4444, "Kgamma": 0x5555,
           "RhoA": 0x6666, "RhoB": 0x7777}
    setup = snark.GenerateTrustedSetup(len(g["witness"]), cc, alphas, betas, gammas, toxic=tox)
    opk, ovk = o.pinocchio_setup(cc["NVars"], cc["NPublic"], alphas, betas, gammas, tox)
    for k in opk:
        assert setup["Pk"][k] == opk[k], k
    for k in ovk:
        assert setup["Vk"][k] == ovk[k], k
    w = [int(x) for x in g["witness"]]
    _, _, _, px = pf.CombinePolynomials(w, alphas, betas, gammas)
    proof = snark.GenerateProofs(cc, setup["Pk"], w, px)
    oproof = o.pinocchio_prove(cc["NVars"], cc["NPublic"], opk, w, px)[0]
    for k, v in oproof.items():
        grp = G2 if k == "PiB" else G1
        assert grp.affine(proof[k]) == grp.affine(v), k
    assert snark.VerifyProof(setup["Vk"], proof, [35], True)
    assert not snark.VerifyProof(setup["Vk"], proof, [34])
    assert o.pinocchio_verify(setup["Vk"], proof, [35])[0]
    # the Go binary's setup and proof (older JSON layout)
    st, pr = g["pinocchio_setup"], g["pinocchio_proofs"]
    t3 = lambda p: tuple(p)
    t2 = lambda p: tuple(tuple(c) for c in p)
    vk = {k: ([t3(p) for p in v] if k == "IC" else (t2(v) if isinstance(v[0], list) else t3(v))) for k, v in st["Vk"].items()}
    gproof = {k: (t2(v) if k == "PiB" else t3(v)) for k, v in pr.items()}
    assert snark.VerifyProof(vk, gproof, [35])
    assert not snark.VerifyProof(vk, gproof, [34])


@pytest.mark.parametrize("kernel", [1, 2])
def test_both_pairing_kernels(mods, golden_dir, kernel):
    """B200_CFG_PAIRING_KERNEL: one thread per pairing (1, the step-by-step restatement) and one warp per pairing (2,
    csrc/pairing_warp.cuh) give the same F_q^12 coefficients: the snarkjs golden (K8), the bn128_test.go literal, the oracle
    on random points and a G1 infinity, and the same errors (G2 infinity, coordinate >= q)."""
    from gosnark_b200 import _lib
    bn, _, _ = mods
    vk, _, _, gold = _circom(golden_dir)
    _lib.check(_lib.lib().b200_config(_lib.CFG_PAIRING_KERNEL, kernel))
    try:
        assert bn.Pairing(vk["G1"]["Alpha"], vk["G2"]["Beta"]) == gold
        rng = random.Random(50 + kernel)
        ps = [G1.mul_scalar(G1.G, 25)] + [G1.mul_scalar(G1.G, rng.randrange(1, R)) for _ in range(5)] + [G1.zero3()]
        qs = [G2.mul_scalar(G2.G, 30)] + [G2.mul_scalar(G2.G, rng.randrange(1, R)) for _ in range(5)] + [G2.G]
        got = bn.PairingBatch(ps, qs)
        assert got[0][0][0][0] == 8016119724813186033542830391460394070015218389456422587891475873290878009957
        for p, q, e in zip(ps, qs, got):
            assert e == o.BN.pairing(p, q)
        with pytest.raises(Exception, match="Fq2.One"):
            bn.Pairing(G1.G, G2.zero3())
        with pytest.raises(Exception, match=">= q"):
            bn.Pairing((o.Q, 2, 1), G2.G)
    finally:
        _lib.check(_lib.lib().b200_config(_lib.CFG_PAIRING_KERNEL, 0))
