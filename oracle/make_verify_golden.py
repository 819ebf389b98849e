#!/usr/bin/env python3
"""Generate tests/golden/gobin_verify_edges.json: the REFERENCE's own prebuilt Go binary (go-snark-cli, see
make_golden.py) verifying crafted Groth16 and Pinocchio proofs at the cases where its verifier's group arithmetic is not
plain group arithmetic.  Test infrastructure only.

    python -m oracle.make_verify_golden      (GOSNARK_REFERENCE overrides where the checkout is looked for)

Two things make the reference's public-input sum differ from the mathematical one (SURVEY H6/H7):
  - bn128 G1.Add has no doubling branch: Add(P, P) is infinity (Z = 0);
  - MulScalar(P, e) walks every bit of |e|, so for |e| >= r a prefix can meet Add(P, P) and restart from infinity.
Every point here is minted from a known discrete log, so the reference's verdict is predictable from the logs alone:
``ic_sum`` below is that model.  Each crafted case comes as two proofs, one valid for the model's sum and one valid for
the mathematical sum; the binary accepts the first and rejects the second.  The file stores the JSON the binary read and
its stdout.  Everything is seeded, so a rerun rewrites the file byte for byte.
"""
import json
import os
import random
import shutil
import subprocess
import sys
import tempfile

from oracle import ref_binary
from oracle import ref_py as o

R = o.R
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "gobin_verify_edges.json")


# ---- the reference's verifier arithmetic on discrete logs (0 = the point at infinity) ------------------------------
def mul_walk(e):
    """m with MulScalar(P, e) == m * P: the double-and-add of bn128/g1.go:140-155 on logs, Add(P, P) -> infinity."""
    e = abs(int(e))
    m = 0
    for i in range(e.bit_length() - 1, -1, -1):
        d = 2 * m % R
        m = (0 if d == 1 else (d + 1) % R) if (e >> i) & 1 else d
    return m


def ref_add(a, b):
    """bn128 G1.Add on logs: infinity is the identity, equal non-zero operands give infinity (no doubling branch)."""
    if a and a == b:
        return 0
    return (a + b) % R


def ic_sum(ic, pubs):
    """icPubl / vkxpia = IC[0] + sum MulScalar(IC[i+1], pubs[i]) in the reference's order (groth16.go:283-286)."""
    acc = ic[0]
    for k, s in zip(ic[1:], pubs):
        acc = ref_add(acc, k * mul_walk(s) % R)
    return acc


def ic_sum_math(ic, pubs):
    return (ic[0] + sum(k * s for k, s in zip(ic[1:], pubs))) % R


def groth16_proof(rng, al, be, ga, de, icp):
    """(a, b, c) with a*b == al*be + icp*ga + c*de: a proof that verifies iff the verifier's icPubl has log icp."""
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    return a, b, (a * b - al * be - icp * ga) * pow(de, -1, R) % R


def groth16_ok(vk, pr, pubs):
    """The reference's verdict from the logs: vk = dict IC, al, be, ga, de; pr = (a, b, c)."""
    a, b, c = pr
    return a * b % R == (vk["al"] * vk["be"] + ic_sum(vk["IC"], pubs) * vk["ga"] + c * vk["de"]) % R


def pinocchio_logs(rng, ic, a, vkx_a):
    """Logs of a Pinocchio vk and a proof with PiA = a that pass all five checks of snark.go:292-372 when the verifier's
    Vkx + PiA has log vkx_a.  Returns (vk, proof) as dicts of logs."""
    r = lambda: rng.randrange(1, R)
    ka, kb, kc, kbg, kg, z, b, h = (r() for _ in range(8))
    c = (vkx_a * b - h * z) % R                                     # check 4: (Vkx + a) b == h z + c
    kp = kbg * (vkx_a + c + b) * pow(kg, -1, R) % R                 # check 5: (Vkx + a + c) kbg + kbg b == kp kg
    vk = {"Vka": ka, "Vkb": kb, "Vkc": kc, "IC": list(ic), "G1Kbg": kbg, "G2Kbg": kbg, "G2Kg": kg, "Vkz": z}
    pr = {"PiA": a, "PiAp": ka * a % R, "PiB": b, "PiBp": kb * b % R, "PiC": c, "PiCp": kc * c % R, "PiH": h, "PiKp": kp}
    return vk, pr


def pinocchio_failed_check(vk, pr, pubs):
    """Index (1..5) of the first of the five checks the reference fails on these logs, 0 when all pass."""
    if pr["PiA"] * vk["Vka"] % R != pr["PiAp"]:
        return 1
    if vk["Vkb"] * pr["PiB"] % R != pr["PiBp"]:
        return 2
    if pr["PiC"] * vk["Vkc"] % R != pr["PiCp"]:
        return 3
    vkx = ic_sum(vk["IC"], pubs)
    if ref_add(vkx, pr["PiA"]) * pr["PiB"] % R != (pr["PiH"] * vk["Vkz"] + pr["PiC"]) % R:
        return 4
    lhs = ref_add(ref_add(vkx, pr["PiA"]), pr["PiC"]) * vk["G2Kbg"] + vk["G1Kbg"] * pr["PiB"]
    if lhs % R != pr["PiKp"] * vk["G2Kg"] % R:
        return 5
    return 0


# ---- logs -> points (oracle double-and-add of the generators; Z != 1 in general) ----------------------------------
G2_KEYS = ("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz", "PiB")


def g1(k):
    return o.BN.G1.mul_scalar(o.BN.G1.G, k)


def g2(k):
    return o.BN.G2.mul_scalar(o.BN.G2.G, k)


def groth16_points(vk, pr):
    v = {"IC": [g1(k) for k in vk["IC"]], "G1": {"Alpha": g1(vk["al"])},
         "G2": {"Beta": g2(vk["be"]), "Gamma": g2(vk["ga"]), "Delta": g2(vk["de"])}}
    return v, {"PiA": g1(pr[0]), "PiB": g2(pr[1]), "PiC": g1(pr[2])}


def pinocchio_points(vk, pr):
    v = {k: ([g1(x) for x in val] if k == "IC" else (g2(val) if k in G2_KEYS else g1(val))) for k, val in vk.items()}
    return v, {k: (g2(val) if k in G2_KEYS else g1(val)) for k, val in pr.items()}


def jl(p):
    """A point as the nested lists Go's encoding/json reads into [3]*big.Int / [3][2]*big.Int."""
    return [list(c) if isinstance(c, (tuple, list)) else c for c in p]


def to_json(obj):
    if isinstance(obj, dict):
        return {k: to_json(v) for k, v in obj.items()}
    if isinstance(obj, list):
        return [jl(p) for p in obj]
    return jl(obj)


# ---- the crafted cases ---------------------------------------------------------------------------------------------
def cases():
    """[(name, kind, vk_json, proof_json, public)]: each crafted case with a model-valid and a math-valid proof."""
    rng = random.Random(20261017)
    out = []
    r = lambda: rng.randrange(1, R)
    # Groth16: non-canonical signals, IC[1] == IC[0] with signal 1, and P + (-P) followed by another term
    g_cases = [("r+2", [r(), r()], [R + 2]),
               ("2r+5", [r(), r()], [2 * R + 5]),
               ("(r+2)*2^7+93", [r(), r()], [((R + 2) << 7) + 93]),
               ("-(r+2)", [r(), r()], [-(R + 2)])]
    k = r()
    g_cases.append(("IC[1]==IC[0], signal 1", [k, k], [1]))
    s, k1 = r(), r()
    g_cases.append(("s*IC[1]==-IC[0], then IC[2]", [(-s * k1) % R, k1, r()], [s, r()]))
    for name, ic, pubs in g_cases:
        vk = {"IC": ic, "al": r(), "be": r(), "ga": r(), "de": r()}
        targets = [("model", ic_sum(ic, pubs))]
        if ic_sum_math(ic, pubs) != targets[0][1]:
            targets.append(("math", ic_sum_math(ic, pubs)))
        for which, icp in targets:
            pr = groth16_proof(rng, vk["al"], vk["be"], vk["ga"], vk["de"], icp)
            pv, pp = groth16_points(vk, pr)
            out.append({"name": f"groth16 {name} / proof for the {which} sum", "kind": "groth16",
                        "vk": {"IC": to_json(pv["IC"]), "G1": {"Alpha": jl(pv["G1"]["Alpha"])},
                               "G2": {x: jl(pv["G2"][x]) for x in ("Beta", "Gamma", "Delta")}},
                        "proof": to_json(pp), "public": pubs, "model_verified": groth16_ok(vk, pr, pubs)})
    # Pinocchio: a signal of r + 2, and Vkx == PiA (Vkx + PiA is infinity by the reference's Add)
    for name, ic, pubs, equal in (("r+2", [r(), r()], [R + 2], False), ("Vkx==PiA", [r(), r()], [r()], True)):
        vkx, vkx_m = ic_sum(ic, pubs), ic_sum_math(ic, pubs)
        a = vkx if equal else r()
        for which, vkx_a in (("model", ref_add(vkx, a)), ("math", (vkx_m + a) % R)):
            vk, pr = pinocchio_logs(rng, ic, a, vkx_a)
            pv, pp = pinocchio_points(vk, pr)
            out.append({"name": f"pinocchio {name} / proof for the {which} sum", "kind": "pinocchio",
                        "vk": {k2: to_json(v) for k2, v in pv.items()}, "proof": to_json(pp), "public": pubs,
                        "model_verified": pinocchio_failed_check(vk, pr, pubs) == 0})
    return out


def run_binary(binary, case):
    """The binary's stdout for `go-snark-cli [groth16] verify` on the case's files, in a scratch directory."""
    d = tempfile.mkdtemp(prefix="gsv_")
    try:
        b = os.path.join(d, "gsc")
        shutil.copy(binary, b)
        os.chmod(b, 0o755)
        # the prebuilt binary also opens compiledcircuit.json (unused by VerifyProof): an empty object will do
        for fname, obj in (("trustedsetup.json", {"Vk": case["vk"]}), ("publicInputs.json", case["public"]),
                           ("proofs.json", case["proof"]), ("compiledcircuit.json", {})):
            with open(os.path.join(d, fname), "w") as f:
                json.dump(obj, f)
        args = ["groth16", "verify"] if case["kind"] == "groth16" else ["verify"]
        p = subprocess.run([b, *args], cwd=d, capture_output=True, text=True, timeout=300)
        return p.stdout + p.stderr
    finally:
        shutil.rmtree(d)


def verdict(stdout):
    """The binary's verdict line (cli/main.go:390-395, 542-547)."""
    if "ERROR: proofs not verified" in stdout:
        return False
    if "Proofs verified" in stdout:
        return True
    raise RuntimeError(f"no verdict in the binary's output:\n{stdout[-2000:]}")


def main():
    ref = ref_binary.require_reference_dir()
    binary = os.path.join(ref, "go-snark-cli")
    gold = cases()
    for c in gold:
        c["go_stdout"] = run_binary(binary, c)
        c["go_verified"] = verdict(c["go_stdout"])
        if c["go_verified"] != c["model_verified"]:
            raise SystemExit(f"{c['name']}: the binary says {c['go_verified']}, the log model {c['model_verified']}")
        print(f"{c['name']}: {'verified' if c['go_verified'] else 'rejected'}")
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0)
        f.write("\n")
    print(len(gold), "cases ->", os.path.normpath(OUT))


if __name__ == "__main__":
    sys.exit(main())
