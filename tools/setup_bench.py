"""Trusted setup from a sparse R1CS, timed: the wall time of b200_groth16_setup and b200_pinocchio_setup on
SyntheticCircuit(2^logn) (host clock around the synchronous call, after a warm-up, median of --reps), beside the two
other ways to get the same key in the same run:
  - minting the same scalars with the reference-order kernel (b200_g1/g2_mul_batch_bcast), one call per group;
  - building CircuitGroth16(logn), which derives the scalars in Python and mints with that kernel.
Each output array is checked on a sample of --sample points against k*G computed on the CPU (oracle/ref_c.c) from the
discrete logs CircuitGroth16 / CircuitPinocchio derive in Python.  Prints one JSON line per size, with the card's name and
power limit.  --profile adds the CUDA time of each setup kernel from torch.profiler (a separate, untimed run).

    python tools/setup_bench.py --logn 16 --logn 20
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gosnark_b200 import _lib, groth16, snark  # noqa: E402
from gosnark_b200._lib import check, ints_to_limbs, lib, limbs_to_ints, ptr  # noqa: E402
from gosnark_b200.bn128 import G1, G2, _flatten_g1, _flatten_g2  # noqa: E402
from gosnark_b200.synthetic import CircuitGroth16, CircuitPinocchio  # noqa: E402
from oracle import ref_py as o  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


def timed(fn, reps):
    fn()                                                   # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts), ts


def bcast(group, k_limbs):
    words = 12 if group == 1 else 24
    out = np.zeros((k_limbs.shape[0], words), dtype=np.uint64)
    gen = _flatten_g1([G1.G]) if group == 1 else _flatten_g2([G2.G])
    fn = lib().b200_g1_mul_batch_bcast if group == 1 else lib().b200_g2_mul_batch_bcast
    return lambda: check(fn(ptr(gen), ptr(k_limbs), k_limbs.shape[0], ptr(out)))


class Checker:
    """k*G on the CPU for a sample of indices, compared with the setup's affine (x, y, 1) points."""

    def __init__(self, sample, seed):
        import build as b200build
        self.oc = ctypes.CDLL(b200build.build_oracle())
        self.threads = self.oc.oc_max_threads()
        self.sample, self.rng = sample, np.random.default_rng(seed)
        self.checked = 0

    def __call__(self, group, pts, dlogs, what):
        pts = np.asarray(pts, dtype=np.uint64).reshape(len(dlogs), -1)
        idx = np.unique(np.concatenate([[0, len(dlogs) - 1], self.rng.integers(0, len(dlogs), self.sample)]))[: self.sample]
        ks = ints_to_limbs([dlogs[i] % o.R for i in idx])
        G = o.BN.G1 if group == 1 else o.BN.G2
        words = 12 if group == 1 else 24
        gen = _flatten_g1([G1.G]) if group == 1 else _flatten_g2([G2.G])
        exp = np.zeros((len(idx), words), dtype=np.uint64)
        fn = self.oc.oc_g1_mul_batch_bcast if group == 1 else self.oc.oc_g2_mul_batch_bcast
        fn(ptr(gen), ptr(ks), ctypes.c_long(len(idx)), self.threads, ptr(exp))
        for j, i in enumerate(idx):
            v = limbs_to_ints(exp[j])
            e = tuple(v) if group == 1 else ((v[0], v[1]), (v[2], v[3]), (v[4], v[5]))
            g = limbs_to_ints(pts[i])
            got = tuple(g) if group == 1 else ((g[0], g[1]), (g[2], g[3]), (g[4], g[5]))
            if G.is_zero(e):
                assert not any(g), (what, int(i))
            else:
                assert got[:2] == tuple(G.affine(e)[:2]) and got[2] == (1 if group == 1 else (1, 0)), (what, int(i))
        self.checked += len(idx)


def profile(run):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    torch.cuda.init()
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        run()
    out = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            out[e.key[:60]] = round(e.device_time_total / 1e3, 3)          # ms
    return dict(sorted(out.items(), key=lambda kv: -kv[1])[:12])


def run(logn, reps, bcast_reps, sample, want_profile):
    n = 1 << logn
    res = {"logn": logn, "n": n}
    t0 = time.perf_counter()
    syn = CircuitGroth16(logn)
    res["circuit_groth16_build_s"] = round(time.perf_counter() - t0, 3)
    m, l1 = syn.m, syn.npublic + 1
    res["m"] = m
    chk = Checker(sample, logn)

    # ---- Groth16
    tox = groth16.toxic_limbs(syn.toxic, groth16.SparseSetup.TOXIC)
    g1 = lambda k: np.zeros((k, 12), dtype=np.uint64)
    g2 = lambda k: np.zeros((k, 24), dtype=np.uint64)
    at, b1, cd, b2, ptd, z, ic = g1(m), g1(m), g1(m), g2(m), g1(m - 1), np.zeros((m - 1, 4), np.uint64), g1(l1)
    a1, be1, d1, be2, ga2, d2 = g1(1), g1(1), g1(1), g2(1), g2(1), g2(1)
    call = lambda: check(lib().b200_groth16_setup(syn.r1cs.handle, syn.npublic, ptr(tox), ptr(at), ptr(b1), ptr(b2), ptr(cd),
                                                  ptr(ptd), ptr(z), ptr(a1), ptr(be1), ptr(d1), ptr(be2), ptr(ga2), ptr(d2), ptr(ic)))
    res["groth16_setup_s"], res["groth16_setup_all_s"] = timed(call, reps)
    k1 = np.concatenate([syn.k_ptd, syn.k_alpha, syn.k_beta, syn.k_delta, syn.k_at, syn.k_b, syn.k_c, ints_to_limbs(syn.k_ic)])
    k2 = np.concatenate([syn.k_b, syn.k_beta, syn.k_gamma, syn.k_delta])
    t1, _ = timed(bcast(1, k1), bcast_reps)
    t2, _ = timed(bcast(2, k2), bcast_reps)
    res["groth16_bcast_s"] = {"g1": t1, "g2": t2, "total": t1 + t2, "g1_points": int(k1.shape[0]), "g2_points": int(k2.shape[0])}
    ti = lambda kl: limbs_to_ints(kl)
    for name, grp, pts, kl in (("At", 1, at, syn.k_at), ("BACGamma1", 1, b1, syn.k_b), ("BACGamma2", 2, b2, syn.k_b),
                               ("BACDelta", 1, cd, syn.k_c), ("PowersTauDelta", 1, ptd, syn.k_ptd)):
        chk(grp, pts, ti(kl), name)
    chk(1, ic, syn.k_ic, "IC")
    tx = syn.toxic
    chk(1, np.concatenate([a1, be1, d1]), [tx["Kalpha"], tx["Kbeta"], tx["Kdelta"]], "Alpha1|Beta1|Delta1")
    chk(2, np.concatenate([be2, ga2, d2]), [tx["Kbeta"], tx["Kgamma"], tx["Kdelta"]], "Beta2|Gamma2|Delta2")
    assert np.array_equal(z, syn.z[: m - 1])
    if want_profile:
        res["groth16_kernels_ms"] = profile(call)

    # ---- Pinocchio
    pin = CircuitPinocchio(n, mint=False)
    k = pin.k
    tox = groth16.toxic_limbs(pin.toxic, snark.SparseSetup.TOXIC)
    arr = {key: g1(m) for key in ("A", "Ap", "Bp", "C", "Cp", "Kp")}
    pb2, g1t, pz, vk1, vk2 = g2(m), g1(m - 1), np.zeros((m - 1, 4), np.uint64), g1(2), g2(5)
    call = lambda: check(lib().b200_pinocchio_setup(pin.r1cs.handle, pin.npublic, ptr(tox), ptr(arr["A"]), ptr(arr["Ap"]),
                                                    ptr(pb2), ptr(arr["Bp"]), ptr(arr["C"]), ptr(arr["Cp"]), ptr(arr["Kp"]),
                                                    ptr(g1t), ptr(pz), ptr(vk1), ptr(vk2)))
    res["pinocchio_setup_s"], res["pinocchio_setup_all_s"] = timed(call, reps)
    vg1, vg2 = ("Vkb", "G1Kbg"), ("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz")
    k1 = ints_to_limbs([x for key in ("A", "Ap", "Bp", "C", "Cp", "Kp", "G1T") for x in k[key]] + [k[v] for v in vg1])
    k2 = ints_to_limbs(k["B"] + [k[v] for v in vg2])
    t1, _ = timed(bcast(1, k1), bcast_reps)
    t2, _ = timed(bcast(2, k2), bcast_reps)
    res["pinocchio_bcast_s"] = {"g1": t1, "g2": t2, "total": t1 + t2, "g1_points": int(k1.shape[0]), "g2_points": int(k2.shape[0])}
    for key in ("A", "Ap", "Bp", "C", "Cp", "Kp"):
        chk(1, arr[key], k[key], key)
    chk(2, pb2, k["B"], "B")
    chk(1, g1t, k["G1T"], "G1T")
    chk(1, vk1, [k[v] for v in vg1], "Vk G1")
    chk(2, vk2, [k[v] for v in vg2], "Vk G2")
    assert np.array_equal(pz, pin.z[: m - 1])
    if want_profile:
        res["pinocchio_kernels_ms"] = profile(call)
    res["points_checked"] = chk.checked
    syn.r1cs.free()
    pin.r1cs.free()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--logn", type=int, action="append", help="log2 of the constraint count (repeatable; default 16 and 20)")
    ap.add_argument("--reps", type=int, default=5, help="timed setup calls per protocol (median reported)")
    ap.add_argument("--bcast-reps", type=int, default=3, help="timed reference-order minting calls per group")
    ap.add_argument("--sample", type=int, default=1024, help="points per output array checked against the CPU")
    ap.add_argument("--profile", action="store_true", help="also report per-kernel CUDA time (torch.profiler)")
    ap.add_argument("--out", help="append the JSON lines to this file")
    a = ap.parse_args()
    _lib.init()
    name, power = card()
    for logn in a.logn or [16, 20]:
        res = {"card": name, "power_limit": power}
        res.update(run(logn, a.reps, a.bcast_reps, a.sample, a.profile))
        line = json.dumps(res)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
