"""CPU: the discrete-log formulas behind CircuitPinocchio (synthetic.pinocchio_key_dlogs / pinocchio_proof_dlogs) against
the oracle's restatement of the reference — snark.GenerateTrustedSetup (snark.go:98-251), snark.GenerateProofs (:254-289)
and snark.VerifyProof (:292-372) — on SyntheticCircuit's dense QAP.  The GPU tests at 2^12..2^16 trust these formulas
for their expectations; this ties them to the reference where the oracle can still run."""
import pytest

from oracle import ref_py as o

G1, G2 = o.BN.G1, o.BN.G2


def kg(group, k):
    return group.affine(group.mul_scalar(group.G, k))


@pytest.mark.parametrize("n", [4, 8])
def test_pinocchio_dlogs_match_oracle_setup_prove_verify(n):
    from gosnark_b200.synthetic import SyntheticCircuit, pinocchio_key_dlogs, pinocchio_proof_dlogs, pinocchio_toxic
    circ = SyntheticCircuit(n)
    alphas, betas, gammas, zpol = o.PF.r1cs_to_qap(*circ.dense())
    tox = pinocchio_toxic()
    t = tox["T"]
    at, bt, ct = ([o.PF.eval(p, t) for p in ps] for ps in (alphas, betas, gammas))
    zt = o.PF.eval(zpol, t)

    pk, vk = o.pinocchio_setup(circ.m, circ.npublic, alphas, betas, gammas, tox)
    k = pinocchio_key_dlogs(at, bt, ct, zt, tox, circ.npublic)
    for s in ("A", "Ap", "Bp", "C", "Cp", "Kp", "G1T"):
        assert len(k[s]) == len(pk[s]), s
        assert [kg(G1, x) for x in k[s]] == [G1.affine(p) for p in pk[s]], s
    assert [kg(G2, x) for x in k["B"]] == [G2.affine(p) for p in pk["B"]]
    for s in ("Vkb", "G1Kbg"):
        assert kg(G1, k[s]) == G1.affine(vk[s]), s
    for s in ("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz"):
        assert kg(G2, k[s]) == G2.affine(vk[s]), s
    assert [kg(G1, x) for x in k["IC"]] == [G1.affine(p) for p in vk["IC"]]

    w = circ.witness
    px = o.PF.combine_polynomials(w, alphas, betas, gammas)[3]
    ref, _ = o.pinocchio_prove(circ.m, circ.npublic, pk, w, px)
    e = pinocchio_proof_dlogs(at, bt, ct, zt, tox, circ.npublic, w)
    assert set(e) == set(ref)
    ours = {s: G1.mul_scalar(G1.G, x) for s, x in e.items() if s != "PiB"}
    ours["PiB"] = G2.mul_scalar(G2.G, e["PiB"])
    for s, p in ref.items():
        grp = G2 if s == "PiB" else G1
        assert grp.affine(ours[s]) == grp.affine(p), s
    assert o.pinocchio_verify(vk, ours, circ.public_signals)[0]
    # the reference binds public signals only through IC = A[0..NPublic]; this circuit's public signal occurs only in C,
    # so IC[1] is the point at infinity and any public value verifies (what the GPU tests rely on)
    assert k["IC"][1] == 0 and o.pinocchio_verify(vk, ours, [circ.public_signals[0] + 1])[0]
