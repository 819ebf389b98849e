"""GPU: the verifier side at benchmark scale and at the reference's degenerate cases.

- b200_pairing_batch on up to 2^16 + 5 pairings, under both kernels and the automatic choice between them, with every
  row compared with an exact value.  Row i is (a_i G1, b_i G2) with a_i b_i = c_k for one of 64 classes c_k, so
  e(P_i, Q_i) = E^(c_k) for E = e(G1, G2): 64 F_q^12 exponentiations on the host check every row.  Negated, rescaled,
  infinite and generator rows sit at random places in every 32-row block.
- groth16.VerifyProof / b200_groth16_verify and snark.VerifyProof on proofs built from known discrete logs.  The expected
  verdict comes from a model of the reference's own sum on the logs (oracle/make_verify_golden.py): Add(P, P) is
  infinity, and MulScalar walks every bit of a non-canonical signal.  Where that sum is not the mathematical one, the
  proof that is valid in plain group arithmetic must be rejected.
- The reference binary's recorded verdicts on the crafted cases (tests/golden/gobin_verify_edges.json), and the binary
  itself when it is staged under oracle/_ref/."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

from arith_edges import base_edges, montgomery_preimages
from oracle import make_verify_golden as mvg
from oracle import ref_py as o

pytestmark = pytest.mark.gpu
R, Q = o.R, o.Q
G1, G2, F2, F12 = o.BN.G1, o.BN.G2, o.BN.Fq2, o.BN.Fq12
EINVAL, ERANGE = -3, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOBIN = os.path.join(ROOT, "oracle", "_ref", "go-snark-cli")


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib


def _u(x):
    return np.frombuffer(int(x).to_bytes(32, "little"), dtype=np.uint64)


def _i(words):
    return int.from_bytes(np.ascontiguousarray(words).tobytes(), "little")


def _f12_limbs(v):
    return np.concatenate([_u(c) for h in v for f2 in h for c in f2])


# ---------------------------------------------------------------------------------------------------------------------
# pairing batches
NMAX = (1 << 16) + 5
PLAIN, NEG, RESCALE, INF, GEN = range(5)
BLOCK_PATTERN = [NEG] * 4 + [RESCALE] * 6 + [INF] * 3 + [GEN] * 2 + [PLAIN] * 17     # one 32-row block


def _lambdas_g1():
    pre = montgomery_preimages(Q, base_edges(Q))
    return [x for x in [2, Q - 1] + pre if x]


def _lambdas_g2():
    pre = montgomery_preimages(Q, base_edges(Q))
    lam = [(0, 1), (Q - 1, Q - 1), (2, 0), (1, Q - 1)] + [(pre[i], pre[-1 - i]) for i in range(len(pre))]
    return [x for x in lam if x != (0, 0)]


@pytest.fixture(scope="module")
def batch(L):
    """NMAX rows: g1 (n, 12) and g2 (n, 24) Jacobian limbs, the expected (n, 48) values, and each row's kind."""
    lib, check, ptr = L.lib, L.check, L.ptr
    rng = random.Random(2026_10_17)
    cs = [1, R - 1] + [rng.randrange(2, R - 1) for _ in range(62)]
    E = o.BN.pairing(G1.G, G2.G)
    pos = [F12.exp(E, c) for c in cs]
    tab_pos = np.stack([_f12_limbs(v) for v in pos])
    tab_neg = np.stack([_f12_limbs(F12.inverse(v)) for v in pos])       # e(-P, Q) = e(P, Q)^-1
    kinds = []
    for _ in range((NMAX + 31) // 32):
        blk = list(BLOCK_PATTERN)
        rng.shuffle(blk)
        kinds += blk
    kinds = np.array(kinds[:NMAX])
    cls = np.array([rng.randrange(len(cs)) for _ in range(NMAX)])
    cls[kinds == GEN] = 0
    a = [rng.randrange(1, R) for _ in range(NMAX)]
    b = [cs[k] * pow(x, -1, R) % R for k, x in zip(cls, a)]
    g1 = np.zeros((NMAX, 12), dtype=np.uint64)
    g2 = np.zeros((NMAX, 24), dtype=np.uint64)
    check(lib().b200_g1_mul_batch_bcast(ptr(L.ints_to_limbs([1, 2, 1])), ptr(L.ints_to_limbs(a)), NMAX, ptr(g1)))
    check(lib().b200_g2_mul_batch_bcast(ptr(L.ints_to_limbs([x for c in G2.G for x in c])), ptr(L.ints_to_limbs(b)),
                                        NMAX, ptr(g2)))
    for i in rng.sample(range(NMAX), 32):       # the minting itself, against the reference's double-and-add
        assert tuple(_i(g1[i, 4 * k:4 * k + 4]) for k in range(3)) == G1.mul_scalar(G1.G, a[i]), i
        want = G2.mul_scalar(G2.G, b[i])
        assert tuple((_i(g2[i, 8 * k:8 * k + 4]), _i(g2[i, 8 * k + 4:8 * k + 8])) for k in range(3)) == want, i
    exp = np.where((kinds == NEG)[:, None], tab_neg[cls], tab_pos[cls])
    lam1, lam2 = _lambdas_g1(), _lambdas_g2()
    q_inf = [G2.G, G2.mul_scalar(G2.G, 7), G2.mul_scalar(G2.G, R - 5)]
    e_inf = [_f12_limbs(o.BN.pairing(G1.zero3(), q)) for q in q_inf]
    q_inf = [np.concatenate([_u(x) for c in q for x in c]) for q in q_inf]
    n_rescaled = 0
    for i in np.nonzero(kinds != PLAIN)[0]:
        k = kinds[i]
        if k == NEG:
            g1[i, 4:8] = _u(Q - _i(g1[i, 4:8]))
        elif k == RESCALE:
            x, y, z = (_i(g1[i, 4 * j:4 * j + 4]) for j in range(3))
            lm = lam1[n_rescaled % len(lam1)]
            g1[i] = np.concatenate([_u(lm * lm * x % Q), _u(lm ** 3 * y % Q), _u(lm * z % Q)])
            x, y, z = ((_i(g2[i, 8 * j:8 * j + 4]), _i(g2[i, 8 * j + 4:8 * j + 8])) for j in range(3))
            lm = lam2[n_rescaled % len(lam2)]
            l2 = F2.square(lm)
            g2[i] = np.concatenate([_u(c) for v in (F2.mul(l2, x), F2.mul(F2.mul(l2, lm), y), F2.mul(lm, z)) for c in v])
            n_rescaled += 1
        elif k == INF:
            if i % 2:
                g1[i] = 0                    # (0, 0, 0)
            else:
                g1[i, 8:12] = 0              # (X, Y, 0) with X, Y != 0: infinity by Z alone, like the reference's IsZero
            j = i % len(q_inf)
            g2[i] = q_inf[j]
            exp[i] = e_inf[j]
        else:
            g1[i] = np.concatenate([_u(1), _u(2), _u(1)])
            g2[i] = np.concatenate([_u(x) for c in G2.G for x in c])
    return {"g1": g1, "g2": g2, "exp": exp, "kinds": kinds}


def _pairing(L, g1, g2, n):
    out = np.zeros((n, 48), dtype=np.uint64)
    rc = L.lib().b200_pairing_batch(L.ptr(np.ascontiguousarray(g1[:n])), L.ptr(np.ascontiguousarray(g2[:n])), n,
                                    L.ptr(out))
    return rc, out


def _assert_rows(got, batch, n):
    bad = np.nonzero((got != batch["exp"][:n]).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} of {n} rows differ; first rows {bad[:8].tolist()}, kinds {batch['kinds'][bad[:8]]}"


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kernel,n", [(0, n) for n in (1, 5, 33, 2047, 2048, 2049, 4099, NMAX)]
                         + [(1, 33), (1, 4099), (2, 33), (2, 4099), (2, NMAX)])
def test_pairing_batch_every_row(L, batch, kernel, n):
    """B200_CFG_PAIRING_KERNEL 0 (auto: one warp per pairing up to 2048, one thread above), 1 (thread) and 2 (warp): every
    row equals its exact value, so the two kernels' outputs are bit-identical too."""
    L.check(L.lib().b200_config(L.CFG_PAIRING_KERNEL, kernel))
    try:
        rc, got = _pairing(L, batch["g1"], batch["g2"], n)
        assert rc == 0, L.lib().b200_last_error().decode()
        _assert_rows(got, batch, n)
    finally:
        L.check(L.lib().b200_config(L.CFG_PAIRING_KERNEL, 0))


@pytest.mark.parametrize("n", [2047, 4099], ids=["warp-kernel", "thread-kernel"])
def test_pairing_batch_errors(L, batch, n):
    """G2 infinity in the last row: B200_EINVAL (the reference panics, bn128.go:238-241); a G1 coordinate equal to q in
    the middle row: B200_ERANGE.  The rows of a failed call are not defined; the next good call is exact."""
    g1, g2 = batch["g1"][:n].copy(), batch["g2"][:n].copy()
    g2[n - 1] = 0
    assert _pairing(L, g1, g2, n)[0] == EINVAL
    g2[n - 1] = batch["g2"][n - 1]
    g1[n // 2, 4 * (n % 3):4 * (n % 3) + 4] = _u(Q)
    assert _pairing(L, g1, g2, n)[0] == ERANGE
    rc, got = _pairing(L, batch["g1"], batch["g2"], n)
    assert rc == 0
    _assert_rows(got, batch, n)


# ---------------------------------------------------------------------------------------------------------------------
# Groth16 verification from known discrete logs
@pytest.fixture(scope="module")
def mint(L):
    from gosnark_b200 import bn128
    g1, g2 = bn128.G1(), bn128.G2()

    def m(group, logs):
        return (g1 if group == 1 else g2).MulScalarBatch([(g1 if group == 1 else g2).G], [int(k) for k in logs])
    return m


def _g16(mint, vk, pr):
    ic = mint(1, vk["IC"])
    a1, pa, pc = mint(1, [vk["al"], pr[0], pr[2]])
    b2, ga, de, pb = mint(2, [vk["be"], vk["ga"], vk["de"], pr[1]])
    return ({"IC": ic, "G1": {"Alpha": a1}, "G2": {"Beta": b2, "Gamma": ga, "Delta": de}},
            {"PiA": pa, "PiB": pb, "PiC": pc})


def _abi_verify(L, vk, proof, pub_limbs, npub):
    """b200_groth16_verify straight from limbs: (rc, ok)."""
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
    ok = ctypes.c_int(-1)
    pub = pub_limbs if npub else np.zeros((1, 4), dtype=np.uint64)
    rc = L.lib().b200_groth16_verify(
        L.ptr(_flatten_g1(vk["IC"])), len(vk["IC"]), L.ptr(_flatten_g1([vk["G1"]["Alpha"]])),
        L.ptr(_flatten_g2([vk["G2"]["Beta"]])), L.ptr(_flatten_g2([vk["G2"]["Gamma"]])),
        L.ptr(_flatten_g2([vk["G2"]["Delta"]])), L.ptr(_flatten_g1([proof["PiA"]])), L.ptr(_flatten_g2([proof["PiB"]])),
        L.ptr(_flatten_g1([proof["PiC"]])), L.ptr(pub), npub, ctypes.byref(ok))
    return rc, ok.value


def _g16_cases():
    """[(name, vk logs, proof logs, public signals)]: proofs for the reference's sum and, where it differs, for the
    mathematical one."""
    rng = random.Random(16)
    r = lambda: rng.randrange(1, R)
    base = []
    for npub in (0, 1, 2, 31, 32, 33, 1000):
        pubs = [rng.choice([0, 1, R - 1, r(), r()]) for _ in range(npub)]
        base.append((f"npub={npub}", [r() for _ in range(npub + 1)], pubs))
    base.append(("3 signals, 6 IC entries", [r() for _ in range(6)], [r(), r(), r()]))
    k = r()
    base.append(("IC[1]==IC[0], signal 1", [k, k], [1]))
    s, k1 = r(), r()
    base.append(("s*IC[1]==IC[0]", [s * k1 % R, k1], [s]))
    s, k1 = r(), r()
    base.append(("s*IC[1]==-IC[0], then more terms", [-s * k1 % R, k1, r(), r()], [s, r(), 0]))
    base.append(("signals 0", [r(), r(), r(), r()], [0, 0, 5]))
    base.append(("IC[0] at infinity", [0, r(), r()], [r(), r()]))
    for label, e in (("r+2", R + 2), ("2r+5", 2 * R + 5), ("(r+2)*2^7+93", ((R + 2) << 7) + 93), ("-(r+2)", -(R + 2))):
        base.append((f"signal {label}", [r(), r(), r()], [r(), e]))
    out = []
    for name, ic, pubs in base:
        vk = {"IC": ic, "al": r(), "be": r(), "ga": r(), "de": r()}
        sums = {"model": mvg.ic_sum(ic, pubs), "math": mvg.ic_sum_math(ic, pubs)}
        for which, icp in sums.items():
            if which == "math" and icp == sums["model"]:
                continue
            out.append((f"{name} / {which}", vk, mvg.groth16_proof(rng, vk["al"], vk["be"], vk["ga"], vk["de"], icp), pubs))
    # valid proofs with PiA or PiC at infinity
    vk = {"IC": [r(), r()], "al": r(), "be": r(), "ga": r(), "de": r()}
    pubs = [r()]
    rhs = (vk["al"] * vk["be"] + mvg.ic_sum(vk["IC"], pubs) * vk["ga"]) % R
    out.append(("PiA at infinity", vk, (0, r(), -rhs * pow(vk["de"], -1, R) % R), pubs))
    a = r()
    out.append(("PiC at infinity", vk, (a, rhs * pow(a, -1, R) % R, 0), pubs))
    return out


G16_CASES = _g16_cases()


@pytest.mark.timeout(600)
def test_groth16_verify_matches_reference_model(L, mint):
    """Every case through groth16.VerifyProof (the Python entry, which maps signals with reduce_scalar) and through
    b200_groth16_verify with the model's reduced signals: both give the reference's verdict.  A proof for the
    mathematical sum is rejected wherever the reference's sum differs (equal operands, non-canonical signals); the
    proof for the reference's sum is accepted, also where the sum passes through P + (-P).  Moving one signal of a
    valid proof rejects it."""
    from gosnark_b200 import groth16
    n_math = 0
    for name, vk, pr, pubs in G16_CASES:
        want = mvg.groth16_ok(vk, pr, pubs)
        assert want == (not name.endswith("/ math")), name
        n_math += name.endswith("/ math")
        pvk, pp = _g16(mint, vk, pr)
        assert groth16.VerifyProof(pvk, pp, pubs) == want, name
        rc, ok = _abi_verify(L, pvk, pp, L.ints_to_limbs([mvg.mul_walk(s) for s in pubs]), len(pubs))
        assert rc == 0 and ok == want, name
        if want and pubs:
            moved = list(pubs)
            moved[-1] = (mvg.mul_walk(moved[-1]) + 1) % R
            assert not mvg.groth16_ok(vk, pr, moved), name
            assert not groth16.VerifyProof(pvk, pp, moved), name
    assert n_math == 6


def test_groth16_verify_proof_points_with_z_not_one(L, mint):
    """The same valid proof with PiA, PiB, PiC rescaled by lambda (Z != 1, edge lambdas): still accepted."""
    from gosnark_b200 import groth16
    name, vk, pr, pubs = G16_CASES[2]
    pvk, pp = _g16(mint, vk, pr)
    assert groth16.VerifyProof(pvk, pp, pubs)
    for l1, l2 in zip(_lambdas_g1()[:6], _lambdas_g2()[:6]):
        x, y, z = pp["PiA"]
        pa = (l1 * l1 * x % Q, l1 ** 3 * y % Q, l1 * z % Q)
        x, y, z = pp["PiC"]
        pc = (l1 * l1 * x % Q, l1 ** 3 * y % Q, l1 * z % Q)
        x, y, z = pp["PiB"]
        sq = F2.square(l2)
        pb = (F2.mul(sq, x), F2.mul(F2.mul(sq, l2), y), F2.mul(l2, z))
        assert groth16.VerifyProof(pvk, {"PiA": pa, "PiB": pb, "PiC": pc}, pubs), (l1, l2)


def test_groth16_model_pinned_to_oracle(mint):
    """The log model against the oracle's restatement of groth16.VerifyProof (groth16.go:281-305) on the cases where
    the reference departs from plain arithmetic."""
    picked = [c for c in G16_CASES if c[0].startswith(("IC[1]==IC[0]", "s*IC[1]==IC[0] / model", "signal r+2 "))]
    assert len(picked) == 5
    for name, vk, pr, pubs in picked:
        pvk, pp = _g16(mint, vk, pr)
        assert o.groth16_verify(pvk, pp, pubs) == mvg.groth16_ok(vk, pr, pubs), name


def test_groth16_verify_errors(L, mint):
    """PiB or a vk G2 point at infinity: B200_EINVAL.  A coordinate >= q: B200_ERANGE.  A signal >= r given to the C ABI:
    B200_ERANGE (the Python entry reduces it first).  A good call afterwards is accepted."""
    name, vk, pr, pubs = G16_CASES[2]
    pvk, pp = _g16(mint, vk, pr)
    sig = L.ints_to_limbs(pubs)
    inf2 = ((0, 0), (0, 0), (0, 0))
    assert _abi_verify(L, pvk, dict(pp, PiB=inf2), sig, len(pubs))[0] == EINVAL
    for k in ("Beta", "Gamma", "Delta"):
        bad = dict(pvk, G2=dict(pvk["G2"], **{k: inf2}))
        assert _abi_verify(L, bad, pp, sig, len(pubs))[0] == EINVAL, k
    x, y, z = pp["PiA"]
    assert _abi_verify(L, pvk, dict(pp, PiA=(Q, y, z)), sig, len(pubs))[0] == ERANGE
    ic = list(pvk["IC"])
    ic[1] = (ic[1][0], ic[1][1] + Q, ic[1][2])
    assert _abi_verify(L, dict(pvk, IC=ic), pp, sig, len(pubs))[0] == ERANGE
    x, y, z = pp["PiB"]
    assert _abi_verify(L, pvk, dict(pp, PiB=(x, y, (z[0], Q))), sig, len(pubs))[0] == ERANGE
    assert _abi_verify(L, pvk, pp, L.ints_to_limbs([pubs[0] + R]), 1)[0] == ERANGE
    assert _abi_verify(L, pvk, pp, sig, len(pubs)) == (0, 1)


# ---------------------------------------------------------------------------------------------------------------------
# Pinocchio verification
def _pin_points(mint, vk, pr):
    g2k = [k for k in vk if k in mvg.G2_KEYS]
    g1k = [k for k in vk if k not in mvg.G2_KEYS and k != "IC"]
    pv = dict(zip(g2k, mint(2, [vk[k] for k in g2k])))
    pv.update(zip(g1k, mint(1, [vk[k] for k in g1k])))
    pv["IC"] = mint(1, vk["IC"])
    prk = [k for k in pr if k != "PiB"]
    pp = dict(zip(prk, mint(1, [pr[k] for k in prk])))
    pp["PiB"] = mint(2, [pr["PiB"]])[0]
    return pv, pp


def _check_lines(golden_dir):
    """The reference's five check lines, as its binary prints them (tests/golden/gobin_x3x5.json)."""
    out = json.load(open(os.path.join(golden_dir, "gobin_x3x5.json")))["pinocchio_verify_stdout"]
    lines = [ln[2:] for ln in out.splitlines() if ln.startswith("✓ ")]
    assert len(lines) == 5
    return lines


@pytest.mark.timeout(600)
def test_pinocchio_verify_each_check(L, mint, capsys, golden_dir):
    """A proof that passes all five checks of snark.VerifyProof (snark.go:292-372), and five variants that each break
    exactly check k.  Each variant is rejected; with debug the output is ✓ for the checks before k and ❌ for check k, and
    k is the index the oracle's restatement returns."""
    from gosnark_b200 import snark
    texts = _check_lines(golden_dir)
    rng = random.Random(55)
    r = lambda: rng.randrange(1, R)
    ic, pubs = [r(), r(), r()], [r(), R - 1]
    a = r()
    vk, pr = mvg.pinocchio_logs(rng, ic, a, mvg.ref_add(mvg.ic_sum(ic, pubs), a))
    pv, pp = _pin_points(mint, vk, pr)
    capsys.readouterr()
    assert snark.VerifyProof(pv, pp, pubs, True)
    assert capsys.readouterr().out.splitlines() == ["✓ " + t for t in texts]
    for k, key in enumerate(("PiAp", "PiBp", "PiCp", "PiH", "PiKp"), start=1):
        bad = dict(pr, **{key: (pr[key] + 1) % R})
        assert mvg.pinocchio_failed_check(vk, bad, pubs) == k
        bv, bp = _pin_points(mint, vk, bad)
        assert not snark.VerifyProof(bv, bp, pubs, True), k
        assert capsys.readouterr().out.splitlines() == ["✓ " + t for t in texts[:k - 1]] + ["❌ " + texts[k - 1]], k
        assert o.pinocchio_verify(bv, bp, pubs) == (False, k)


@pytest.mark.timeout(600)
def test_pinocchio_verify_reference_sums(L, mint):
    """Vkx == PiA (Vkx + PiA is infinity by the reference's Add) and a public signal of r + 2: the proof for the
    reference's sum is accepted and the one for the mathematical sum is rejected, like the log model; the oracle agrees
    on two of them."""
    from gosnark_b200 import snark
    rng = random.Random(56)
    r = lambda: rng.randrange(1, R)
    runs = []
    for name, ic, pubs, equal in (("Vkx==PiA", [r(), r()], [r()], True), ("r+2", [r(), r()], [R + 2], False)):
        vkx, vkx_m = mvg.ic_sum(ic, pubs), mvg.ic_sum_math(ic, pubs)
        a = vkx if equal else r()
        for which, vkx_a in (("model", mvg.ref_add(vkx, a)), ("math", (vkx_m + a) % R)):
            vk, pr = mvg.pinocchio_logs(rng, ic, a, vkx_a)
            want = mvg.pinocchio_failed_check(vk, pr, pubs)
            assert (want == 0) == (which == "model"), (name, which)
            pv, pp = _pin_points(mint, vk, pr)
            assert snark.VerifyProof(pv, pp, pubs) == (want == 0), (name, which)
            runs.append((name, which, pv, pp, pubs, want))
    for name, which, pv, pp, pubs, want in (runs[0], runs[3]):
        assert o.pinocchio_verify(pv, pp, pubs) == (want == 0, want), (name, which)


# ---------------------------------------------------------------------------------------------------------------------
# the reference binary's verdicts
def _load_case(c):
    t3 = lambda p: tuple(int(x) for x in p)
    t2 = lambda p: tuple(tuple(int(x) for x in q) for q in p)
    if c["kind"] == "groth16":
        v = c["vk"]
        vk = {"IC": [t3(p) for p in v["IC"]], "G1": {"Alpha": t3(v["G1"]["Alpha"])},
              "G2": {k: t2(v["G2"][k]) for k in ("Beta", "Gamma", "Delta")}}
    else:
        vk = {k: ([t3(p) for p in v] if k == "IC" else (t2(v) if k in mvg.G2_KEYS else t3(v))) for k, v in c["vk"].items()}
    proof = {k: (t2(v) if k == "PiB" else t3(v)) for k, v in c["proof"].items()}
    return vk, proof


@pytest.fixture(scope="module")
def gobin_cases(golden_dir):
    return json.load(open(os.path.join(golden_dir, "gobin_verify_edges.json")))


@pytest.mark.timeout(900)
def test_device_verdict_equals_go_binary(L, gobin_cases):
    """For each crafted case of gobin_verify_edges.json, the device verdict equals the one `go-snark-cli [groth16]
    verify` recorded; the binary, when staged, still gives it."""
    from gosnark_b200 import groth16, snark
    assert len(gobin_cases) == 15 and sum(c["go_verified"] for c in gobin_cases) == 8
    for c in gobin_cases:
        vk, proof = _load_case(c)
        ver = groth16.VerifyProof if c["kind"] == "groth16" else snark.VerifyProof
        assert ver(vk, proof, c["public"]) == c["go_verified"], c["name"]
        if os.path.exists(GOBIN):
            assert mvg.verdict(mvg.run_binary(GOBIN, c)) == c["go_verified"], c["name"]


def test_cli_verify_prints_go_output(L, gobin_cases, tmp_path, monkeypatch, capsys):
    """`cli groth16 verify` and `cli verify` (Pinocchio) on each case's files print what the Go CLI printed: the
    verdict and the ✓/❌ check lines, for a public input of r + 2 among others."""
    from gosnark_b200 import cli
    monkeypatch.chdir(tmp_path)
    for c in gobin_cases:
        for fname, obj in (("trustedsetup.json", {"Vk": c["vk"]}), ("publicInputs.json", c["public"]),
                           ("proofs.json", c["proof"])):
            with open(fname, "w") as f:
                json.dump(obj, f)
        capsys.readouterr()
        assert cli.main(["groth16", "verify"] if c["kind"] == "groth16" else ["verify"]) == 0
        assert capsys.readouterr().out.splitlines() == c["go_stdout"].splitlines(), c["name"]
