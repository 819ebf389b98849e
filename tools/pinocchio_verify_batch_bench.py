#!/usr/bin/env python3
"""Batched Pinocchio verification timed against its alternatives (development aid; bench.py is the contract).

CircuitPinocchio at 2^12 constraints: 64 proofs of distinct satisfying witnesses made by one
b200_pinocchio_prove_witness_batch_device call, tiled to k proofs.  For each k in --ks, ms per proof of
  - b200_pinocchio_verify_batch_device on the prover's layout, under B200_CFG_PAIRING_KERNEL 0 (auto), 1 (a thread per
    Miller loop) and 2 (a warp per Miller loop), CUDA events over --steps calls after --warmup, with whether status bit 1
    (the per-proof check ran) stayed clear and every verdict was 1;
  - (a) k calls of snark.VerifyProof (at most --single-cap calls timed, the mean extrapolated);
  - (b) the 12k pairings of the same proofs through one b200_pairing_batch call (host wall time, synchronous entry).
The card's name and power limit are part of the numbers.  Prints one JSON line."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gosnark_b200 import _lib, bn128, snark  # noqa: E402
from gosnark_b200._lib import check, ints_to_limbs, ptr  # noqa: E402
from gosnark_b200.bn128 import _flatten_g1, _flatten_g2, _unflatten_g1, _unflatten_g2  # noqa: E402
from gosnark_b200.synthetic import CircuitPinocchio, SyntheticCircuit  # noqa: E402

ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def events_ms(fn, stream, warmup, steps):
    """ms per call of fn, which queues its work on `stream` (a torch.cuda.Stream)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def g1_add(p, q):
    out = np.zeros(12, np.uint64)
    check(_lib.lib().b200_g1_add_batch(ptr(np.ascontiguousarray(p)), ptr(np.ascontiguousarray(q)), 1, ptr(out)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logn", type=int, default=12)
    ap.add_argument("--ks", default="1,8,64,512,4096")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--single-cap", type=int, default=16)
    args = ap.parse_args()
    _lib.init(0)
    L = _lib.lib()
    n, base = 1 << args.logn, 64
    syn = CircuitPinocchio(n)
    pk = syn.load_pk()
    cs = [SyntheticCircuit(n, seed=0xB1CC + p) for p in range(base)]
    d_w = torch.from_numpy(ints_to_limbs([v for c in cs for v in c.witness]).reshape(-1).view(np.int64)).cuda()
    d_out = torch.zeros(108 * base, dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()                          # the device entry queues on the stream the events time
    st = stream.cuda_stream                               # (never the legacy default stream: its handle is NULL)
    check(L.b200_pinocchio_prove_witness_batch_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, base, d_out.data_ptr(), st))
    torch.cuda.synchronize()
    words = d_out.cpu().numpy().view(np.uint64).reshape(base, 108).copy()
    proofs = []
    for w in words:
        p = dict(zip(ORDER, _unflatten_g1(w[:84])))
        p["PiB"] = _unflatten_g2(w[84:])[0]
        proofs.append(p)
    pubs = [c.public_signals for c in cs]
    vk = syn.vk
    ic = _flatten_g1(vk["IC"])
    vk_g1 = _flatten_g1([vk["Vkb"], vk["G1Kbg"]])
    vk_g2 = _flatten_g2([vk["Vka"], vk["Vkc"], vk["G2Kbg"], vk["G2Kg"], vk["Vkz"]])
    out = {"workload": "pinocchio_verify_batch", "n": n, "gpu": card()[0], "power_limit": card()[1], "k": {}}
    # S and T of every proof for the pairing-batch comparison, by the library's own scalar product and addition
    ic_w = ic.reshape(-1, 12)
    pairs1, pairs2 = [], []
    g2g, vka, vkc, g2kbg, g2kg, vkz = (_flatten_g2([q]).reshape(-1) for q in
                                       (bn128.G2().G, vk["Vka"], vk["Vkc"], vk["G2Kbg"], vk["G2Kg"], vk["Vkz"]))
    vkb, g1kbg = (_flatten_g1([q]).reshape(-1) for q in (vk["Vkb"], vk["G1Kbg"]))
    for p, w in enumerate(words):
        t = np.zeros(12, np.uint64)
        check(L.b200_g1_mul_batch(ptr(np.ascontiguousarray(ic_w[1])), ptr(ints_to_limbs(pubs[p])), 1, ptr(t)))
        s_ = g1_add(g1_add(ic_w[0], t), w[0:12])
        t_ = g1_add(s_, w[36:48])
        g = lambda slot: w[12 * slot:12 * slot + 12]
        pb = w[84:108]
        pairs1.append(np.concatenate([g(0), g(1), vkb, g(2), g(3), g(4), s_, g(5), g(3), t_, g1kbg, g(6)]))
        pairs2.append(np.concatenate([vka, g2g, pb, g2g, vkc, g2g, pb, vkz, g2g, g2kbg, pb, g2kg]))
    rng = random.Random(1)
    for k in [int(x) for x in args.ks.split(",")]:
        reps = (k + base - 1) // base
        d_proofs = d_out.view(base, 108).repeat(reps, 1)[:k].reshape(-1).contiguous()
        d_pub = torch.from_numpy(ints_to_limbs([s for ps in (pubs * reps)[:k] for s in ps]).reshape(-1).view(np.int64)).cuda()
        rho = np.array([rng.randrange(1, 1 << 64) for _ in range(10 * k)], dtype=np.uint64)
        d_ok = torch.zeros(k + 1, dtype=torch.int32, device="cuda")
        row = {}
        for kern, name in ((0, "auto"), (1, "thread"), (2, "warp")):
            check(L.b200_config(_lib.CFG_PAIRING_KERNEL, kern))
            run = lambda: check(L.b200_pinocchio_verify_batch_device(ptr(ic), len(vk["IC"]), ptr(vk_g1), ptr(vk_g2),
                                                                     d_proofs.data_ptr(), d_pub.data_ptr(), 1, k, ptr(rho),
                                                                     d_ok.data_ptr(), st))
            ms = events_ms(run, stream, args.warmup, args.steps)
            res = d_ok.cpu().numpy()
            row[name] = {"ms_per_proof": round(ms / k, 5), "all_ok": bool((res[:k] == 1).all()),
                         "per_proof_path_clear": not (int(res[k]) & 2), "status": int(res[k])}
        check(L.b200_config(_lib.CFG_PAIRING_KERNEL, 0))
        # (a) single calls of snark.VerifyProof
        cnt = min(k, args.single_cap)
        snark.VerifyProof(vk, proofs[0], pubs[0])                                        # warm-up
        t0 = time.perf_counter()
        for p in range(cnt):
            assert snark.VerifyProof(vk, proofs[p % base], pubs[p % base])
        row["single_verify_ms_per_proof"] = round((time.perf_counter() - t0) * 1e3 / cnt, 4)
        # (b) 12k pairings in one b200_pairing_batch call
        g1s = np.concatenate([pairs1[p % base] for p in range(k)])
        g2s = np.concatenate([pairs2[p % base] for p in range(k)])
        po = np.zeros(48 * 12 * k, np.uint64)
        check(L.b200_pairing_batch(ptr(g1s), ptr(g2s), 12 * k, ptr(po)))            # warm-up
        t0 = time.perf_counter()
        check(L.b200_pairing_batch(ptr(g1s), ptr(g2s), 12 * k, ptr(po)))
        row["pairing_batch_12k_ms_per_proof"] = round((time.perf_counter() - t0) * 1e3 / k, 5)
        out["k"][str(k)] = row
    check(L.b200_pk_free(pk))
    print(json.dumps(out))
    ok = all(r[v]["all_ok"] and r[v]["per_proof_path_clear"] for r in out["k"].values() for v in ("auto", "thread", "warp"))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
