#!/usr/bin/env python3
"""Generate tests/golden/*.json by running the REFERENCE's own prebuilt Go
binary (go-snark-cli at the root of the reference tree, built by build-cli.sh:3-4 from
cli/main.go).  Test infrastructure only.

Run where a checkout of the reference exists:
    python oracle/make_golden.py      (GOSNARK_REFERENCE overrides where the checkout is looked for, oracle/ref_binary.py)

For each circuit it runs, in a scratch dir, the CLI workflow of
cli/main.go:28-78:
    compile <circuit>           -> compiledcircuit.json, px.json  (+ stdout: witness, R1CS, QAP)
    trustedsetup / genproofs / verify                 (Pinocchio, snark.go)
    groth16 trustedsetup / genproofs / verify         (groth16/groth16.go)
and stores the JSON files verbatim plus the parsed witness.  Pinocchio
GenerateProofs is deterministic (snark.go:254-289) so its proofs.json is a
bit-exact golden for the whole prove path incl. Jacobian coordinates; Groth16
draws r,s from crypto/rand (groth16.go:231-238) so its proofs.json is only a
golden for the verifier.
"""
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

import ref_binary

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")

CIRCUITS = {
    # config 1: groth16/groth16_test.go:20-28 (flat form)
    "x3x5": dict(
        code="func main(private s0, public s1):\n\ts2 = s0 * s0\n\ts3 = s2 * s0\n\ts4 = s3 + s0\n"
             "\ts5 = s4 + 5\n\tequals(s1, s5)\n\tout = 1 * 1\n",
        private=[3], public=[35]),
    # snark_test.go:245-262 style multiplication circuit (n=4 constraints)
    "mul": dict(
        code="func main(private a, private b, public c):\n\td = a * b\n\tequals(c, d)\n\tout = 1 * 1\n",
        private=[3, 11], public=[33]),
    # largest size at which the reference's R1CSToQAP is correct (21 constraints, SURVEY E3)
    "chain21": dict(
        code="func main(private s0, public s1):\n\tm0 = s0 * s0\n"
             + "".join(f"\tm{i} = m{i-1} * s0\n" for i in range(1, 18))
             + "\tequals(s1, m17)\n\tout = 1 * 1\n",
        private=[2], public=[2 ** 19]),
}


def run(binary, cwd, *args):
    p = subprocess.run([binary, *args], cwd=cwd, capture_output=True, text=True, timeout=120)
    if p.returncode != 0:
        raise RuntimeError(f"{args}: rc={p.returncode}\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
    return p.stdout


def load(path):
    with open(path) as f:
        return json.load(f)


def main():
    ref = ref_binary.require_reference_dir()
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="gsc_")
    binary = os.path.join(tmp, "gsc")
    shutil.copy(os.path.join(ref, "go-snark-cli"), binary)
    os.chmod(binary, 0o755)
    for name, c in CIRCUITS.items():
        d = os.path.join(tmp, name)
        os.makedirs(d)
        with open(os.path.join(d, "test.circuit"), "w") as f:
            f.write(c["code"])
        with open(os.path.join(d, "privateInputs.json"), "w") as f:
            json.dump(c["private"], f)
        with open(os.path.join(d, "publicInputs.json"), "w") as f:
            json.dump(c["public"], f)
        out = run(binary, d, "compile", "test.circuit")
        m = re.search(r"witness \[([^\]]*)\]", out)
        witness = [int(x) for x in m.group(1).split()]
        gold = {"name": name, "circuit_code": c["code"], "private": c["private"], "public": c["public"],
                "witness": witness, "compile_stdout": out,
                "compiledcircuit": load(os.path.join(d, "compiledcircuit.json")),
                "px": load(os.path.join(d, "px.json"))}
        # Pinocchio
        run(binary, d, "trustedsetup")
        gold["pinocchio_setup"] = load(os.path.join(d, "trustedsetup.json"))
        out = run(binary, d, "genproofs")
        gold["pinocchio_proofs"] = load(os.path.join(d, "proofs.json"))
        gold["pinocchio_genproofs_stdout"] = out
        gold["pinocchio_verify_stdout"] = run(binary, d, "verify")
        # Groth16
        run(binary, d, "groth16", "trustedsetup")
        gold["groth16_setup"] = load(os.path.join(d, "trustedsetup.json"))
        out = run(binary, d, "groth16", "genproofs")
        gold["groth16_proofs"] = load(os.path.join(d, "proofs.json"))
        gold["groth16_genproofs_stdout"] = out
        gold["groth16_verify_stdout"] = run(binary, d, "groth16", "verify")
        with open(os.path.join(OUT, f"gobin_{name}.json"), "w") as f:
            json.dump(gold, f)
        print(name, "witness", witness, "ok;", len(json.dumps(gold)), "bytes")
    shutil.rmtree(tmp)
    # K8: the snarkjs-generated Groth16 fixture the reference verifies in
    # externalVerif/circomVerifier_test.go:9-13 (data files, stored verbatim).
    cdir = os.path.join(ref, "externalVerif", "circom-test")
    circom = {k: load(os.path.join(cdir, f)) for k, f in
              (("vk", "verification_key.json"), ("proof", "proof.json"), ("public", "public.json"))}
    with open(os.path.join(OUT, "circom_groth16.json"), "w") as f:
        json.dump(circom, f)
    print("circom fixture ok")


if __name__ == "__main__":
    sys.exit(main())
