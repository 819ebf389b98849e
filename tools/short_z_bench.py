#!/usr/bin/env python3
"""Witness-fed proving on circuits with m = n + 1 signals (len(Z) = n) next to m = n + 2 at the same n, both protocols
(development aid; bench.py is the contract).

For each protocol, size and shape: synthetic.CircuitGroth16 / CircuitPinocchio (``short_z`` for m = n + 1), one key per
prove context on one resident R1CS.  Measured from device memory with CUDA events: ms per device witness-fed proof one at
a time and two in flight (the context-1 key on a second stream), at every --single-logn; ms per proof of
batches of --k witnesses (b200_*_prove_witness_batch_device) at every --batch-logn.  The first and the last timed proof
of each point are checked against their known discrete logs (Groth16: the instance's r, s); a mismatch makes the script
exit non-zero.  --lib PATH times another build of the library (e.g. the parent commit's, in an ignored path of the tree)
from the same Python, so two builds can be compared in one session.  Prints one JSON line with the card's name and power
limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gosnark_b200 import _lib  # noqa: E402
from gosnark_b200._lib import check, ints_to_limbs, ptr  # noqa: E402
from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2  # noqa: E402
from gosnark_b200.synthetic import CircuitGroth16, CircuitPinocchio  # noqa: E402
from oracle import ref_py as o  # noqa: E402

G1, G2 = o.BN.G1, o.BN.G2
PIN_ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


def card():
    """Name and power limit of device 0, read now (the limit is part of every number measured on it)."""
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_ms(run, count, streams, warmup, steps):
    """ms per proof: run(j, stream) issues one proof / batch on stream j; one event pair brackets all steps."""
    for i in range(warmup * len(streams)):
        run(i % len(streams), streams[i % len(streams)])
    torch.cuda.synchronize()
    e0, e1, e_side = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record(streams[0])
    for st in streams[1:]:
        st.wait_event(e0)
    for i in range(steps * len(streams)):
        run(i % len(streams), streams[i % len(streams)])
    for st in streams[1:]:
        e_side.record(st)
        streams[0].wait_event(e_side)
    e1.record(streams[0])
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (steps * len(streams) * count)


def g16_ok(syn, words):
    a, c, b = (np.ascontiguousarray(x) for x in (words[:12], words[12:24], words[24:48]))
    ea, eb, ec = syn.expected_dlogs()
    return (G1.affine(_unflatten_g1(a)[0]) == G1.affine(G1.mul_scalar(G1.G, ea))
            and G2.affine(_unflatten_g2(b)[0]) == G2.affine(G2.mul_scalar(G2.G, eb))
            and G1.affine(_unflatten_g1(c)[0]) == G1.affine(G1.mul_scalar(G1.G, ec)))


def pin_ok(syn, words):
    d = syn.expected_dlogs()
    g1 = _unflatten_g1(np.ascontiguousarray(words[:84]))
    pb = _unflatten_g2(np.ascontiguousarray(words[84:108]))[0]
    return (all(G1.affine(p) == G1.affine(G1.mul_scalar(G1.G, d[k])) for p, k in zip(g1, PIN_ORDER))
            and G2.affine(pb) == G2.affine(G2.mul_scalar(G2.G, d["PiB"])))


def bench_point(L, proto, n, short, ks, args):
    syn = (CircuitGroth16 if proto == "groth16" else CircuitPinocchio)(n=n, short_z=short)
    pks = []
    try:
        for ctx in range(2):
            check(L.b200_config(_lib.CFG_PK_CONTEXT, ctx))
            pks.append(syn.load_pk())
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))
    h, m = syn.r1cs.handle, syn.m
    words = 48 if proto == "groth16" else 108
    ok_fn = g16_ok if proto == "groth16" else pin_ok
    kmax = max(ks) if ks else 1
    d_w = torch.from_numpy(np.tile(syn.w, (kmax, 1)).reshape(-1).view(np.int64)).cuda()
    r_l, s_l = (ints_to_limbs([getattr(syn, a, 0)] * kmax) for a in ("r", "s"))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    out = torch.zeros(words * kmax, dtype=torch.int64, device="cuda")
    outs1 = [torch.zeros(words, dtype=torch.int64, device="cuda") for _ in range(2)]
    res = {"protocol": proto, "n": n, "m": m, "len_Z": int(syn.z.shape[0])}
    bad = []

    def single(c, st):
        if proto == "groth16":
            check(L.b200_groth16_prove_witness_device(pks[c], h, d_w.data_ptr(), m, ptr(r_l), ptr(s_l), outs1[c].data_ptr(),
                                                      st.cuda_stream))
        else:
            check(L.b200_pinocchio_prove_witness_device(pks[c], h, d_w.data_ptr(), m, outs1[c].data_ptr(), st.cuda_stream))

    def checked(name, arr, cnt):
        torch.cuda.synchronize()
        raw = arr.cpu().numpy().view(np.uint64)
        for p in sorted({0, cnt - 1}):
            if not ok_fn(syn, raw[words * p:words * (p + 1)]):
                bad.append(f"{name}[{p}]")

    if n in args.single_n:
        res["single_one_at_a_time_ms"] = round(time_ms(single, 1, streams[:1], args.warmup, args.steps), 4)
        checked("single", outs1[0], 1)
        res["single_two_in_flight_ms"] = round(time_ms(single, 1, streams, args.warmup, args.steps), 4)
        checked("single-ctx0", outs1[0], 1)
        checked("single-ctx1", outs1[1], 1)
    for k in ks:
        def batch(_, st, k=k):
            if proto == "groth16":
                check(L.b200_groth16_prove_witness_batch_device(pks[0], h, d_w.data_ptr(), m, k, ptr(r_l), ptr(s_l),
                                                                out.data_ptr(), st.cuda_stream))
            else:
                check(L.b200_pinocchio_prove_witness_batch_device(pks[0], h, d_w.data_ptr(), m, k, out.data_ptr(), st.cuda_stream))
        res[f"batch_k{k}_ms_per_proof"] = round(time_ms(batch, k, streams[:1], args.warmup, args.steps), 4)
        checked(f"batch{k}", out, k)
    res["bad_proofs"] = bad
    for pk in pks:
        check(L.b200_pk_free(pk))
    syn.r1cs.free()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--single-logn", type=int, nargs="*", default=[12, 16, 20])
    ap.add_argument("--batch-logn", type=int, nargs="*", default=[12, 16])
    ap.add_argument("--k", type=int, nargs="*", default=[1, 8, 64])
    ap.add_argument("--protocols", nargs="+", default=["groth16", "pinocchio"], choices=["groth16", "pinocchio"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", help="time this build of libb200snark.so instead of the tree's")
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 1 or (args.k and min(args.k) < 1):
        ap.error("--steps, --warmup and every k must be >= 1")
    if not torch.cuda.is_available():
        raise SystemExit("short_z_bench: no CUDA device (the library has no CPU fallback)")
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    _lib.init(0)
    L = _lib.lib()
    args.single_n = {1 << x for x in args.single_logn}
    batch_n = {1 << x for x in args.batch_logn}
    points = []
    for proto in args.protocols:
        for n in sorted(args.single_n | batch_n):
            for short in (True, False):
                points.append(bench_point(L, proto, n, short, sorted(set(args.k)) if n in batch_n else [], args))
    name, power = card()
    ok = all(not p["bad_proofs"] for p in points)
    print(json.dumps({"workload": "witness-fed proving, m = n + 1 (len(Z) = n) next to m = n + 2", "lib": _lib.LIB_PATH,
                      "gpu": name, "power_limit": power, "steps": args.steps, "warmup": args.warmup, "points": points,
                      "ok": ok}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
