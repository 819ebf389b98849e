#!/usr/bin/env python3
"""Batched Groth16 verification timed against its alternatives (development aid; bench.py is the contract).

CircuitGroth16 at 2^12 constraints: 64 proofs of distinct satisfying witnesses made by one
b200_groth16_prove_witness_batch_device call, tiled to k proofs.  For each k in --ks, ms per proof of
  - b200_groth16_verify_batch_device on the prover's layout, under B200_CFG_PAIRING_KERNEL 0 (auto), 1 (a thread per
    Miller loop) and 2 (a warp per Miller loop), CUDA events over --steps calls after --warmup, with whether status bit 1
    (the per-proof check ran) stayed clear and every verdict was 1;
  - (a) k calls of b200_groth16_verify (at most --single-cap calls timed, the mean extrapolated);
  - (b) the 4k pairings of the same proofs through one b200_pairing_batch call (host wall time, synchronous entry);
  - (c) the batch prover's ms per proof at 2^12 with k = 64.
The card's name and power limit are part of the numbers.  Prints one JSON line."""
import argparse
import ctypes
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gosnark_b200 import _lib  # noqa: E402
from gosnark_b200._lib import check, ints_to_limbs, ptr  # noqa: E402
from gosnark_b200.synthetic import CircuitGroth16, SyntheticCircuit  # noqa: E402

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


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
    syn = CircuitGroth16(n=n)
    pk = syn.load_pk()
    cs = [SyntheticCircuit(n, seed=0xBE7C + p) for p in range(base)]
    rng = random.Random(1)
    rs, ss = ints_to_limbs([rng.randrange(1, R) for _ in range(base)]), ints_to_limbs([rng.randrange(1, R) for _ in range(base)])
    d_w = torch.from_numpy(ints_to_limbs([v for c in cs for v in c.witness]).reshape(-1).view(np.int64)).cuda()
    d_out = torch.zeros(48 * base, dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()                          # both device entries queue on the stream the events time
    st = stream.cuda_stream                               # (never the legacy default stream: its handle is NULL)
    prove = lambda: check(L.b200_groth16_prove_witness_batch_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, base, ptr(rs),
                                                                    ptr(ss), d_out.data_ptr(), st))
    prove_ms = events_ms(prove, stream, 1, 3) / base
    words = d_out.cpu().numpy().view(np.uint64).reshape(base, 48).copy()
    pubs = [c.public_signals[0] for c in cs]
    ic, a1, b2, g2, d2 = syn.vk_limbs()
    npub = 1
    out = {"workload": "groth16_verify_batch", "n": n, "gpu": card()[0], "power_limit": card()[1],
           "prove_batch64_ms_per_proof": round(prove_ms, 4), "k": {}}
    # icPubl for the pairing-batch comparison: IC[0] + s IC[1] by the library's own scalar product and addition
    icp = []
    for s in pubs:
        t = np.zeros(12, np.uint64)
        check(L.b200_g1_mul_batch(ptr(np.ascontiguousarray(ic[1])), ptr(ints_to_limbs([s])), 1, ptr(t)))
        u = np.zeros(12, np.uint64)
        check(L.b200_g1_add_batch(ptr(np.ascontiguousarray(ic[0])), ptr(t), 1, ptr(u)))
        icp.append(u)
    for k in [int(x) for x in args.ks.split(",")]:
        reps = (k + base - 1) // base
        d_proofs = d_out.view(base, 48).repeat(reps, 1)[:k].reshape(-1).contiguous()
        d_pub = torch.from_numpy(ints_to_limbs((pubs * reps)[:k]).reshape(-1).view(np.int64)).cuda()
        rho = np.array([rng.randrange(1, 1 << 64) for _ in range(2 * k)], dtype=np.uint64)
        d_ok = torch.zeros(k + 1, dtype=torch.int32, device="cuda")
        row = {}
        for kern, name in ((0, "auto"), (1, "thread"), (2, "warp")):
            check(L.b200_config(_lib.CFG_PAIRING_KERNEL, kern))
            run = lambda: check(L.b200_groth16_verify_batch_device(ptr(ic), ic.shape[0], ptr(a1), ptr(b2), ptr(g2), ptr(d2),
                                                                   d_proofs.data_ptr(), d_pub.data_ptr(), npub, k, ptr(rho),
                                                                   d_ok.data_ptr(), st))
            ms = events_ms(run, stream, args.warmup, args.steps)
            res = d_ok.cpu().numpy()
            row[name] = {"ms_per_proof": round(ms / k, 5), "all_ok": bool((res[:k] == 1).all()),
                         "per_proof_path_clear": not (int(res[k]) & 2), "status": int(res[k])}
        check(L.b200_config(_lib.CFG_PAIRING_KERNEL, 0))
        # (a) single calls
        cnt = min(k, args.single_cap)
        okc = ctypes.c_int(0)
        t0 = time.perf_counter()
        for p in range(cnt):
            w = words[p % base]
            check(L.b200_groth16_verify(ptr(ic), ic.shape[0], ptr(a1), ptr(b2), ptr(g2), ptr(d2), ptr(np.ascontiguousarray(w[:12])),
                                        ptr(np.ascontiguousarray(w[24:48])), ptr(np.ascontiguousarray(w[12:24])),
                                        ptr(ints_to_limbs([pubs[p % base]])), 1, ctypes.byref(okc)))
        row["single_verify_ms_per_proof"] = round((time.perf_counter() - t0) * 1e3 / cnt, 4)
        # (b) 4k pairings in one b200_pairing_batch call
        g1s = np.concatenate([np.concatenate([words[p % base][:12], a1.reshape(-1), icp[p % base], words[p % base][12:24]])
                              for p in range(k)])
        g2s = np.concatenate([np.concatenate([words[p % base][24:48], b2.reshape(-1), g2.reshape(-1), d2.reshape(-1)])
                              for p in range(k)])
        po = np.zeros(48 * 4 * k, np.uint64)
        check(L.b200_pairing_batch(ptr(g1s), ptr(g2s), 4 * k, ptr(po)))            # warm-up
        t0 = time.perf_counter()
        check(L.b200_pairing_batch(ptr(g1s), ptr(g2s), 4 * k, ptr(po)))
        row["pairing_batch_4k_ms_per_proof"] = round((time.perf_counter() - t0) * 1e3 / k, 5)
        out["k"][str(k)] = row
    check(L.b200_pk_free(pk))
    print(json.dumps(out))
    ok = all(r[v]["all_ok"] and r[v]["per_proof_path_clear"] for r in out["k"].values() for v in ("auto", "thread", "warp"))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
