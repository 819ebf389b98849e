#!/usr/bin/env python3
"""Batched witness-fed Groth16 proving timed from device memory (development aid; bench.py is the contract).

CircuitGroth16(logn) for each --logn: a real CRS with known discrete logs, one key and one resident R1CS.  For each k,
b200_groth16_prove_witness_batch_device proves k distinct satisfying witnesses (SyntheticCircuit(n, seed=...)) with
distinct (r, s); ms per proof from CUDA events over whole batches.  Beside them, the single witness-fed device proof one
at a time and with two in flight (a second key on prove context 1, as tools/witness_prove_bench.py measures it), the
key's b200_pk_device_bytes after the largest batch, and the card's name and power limit.  --max-gib skips the (n, k)
points whose batch scratch, extrapolated from the k = 1 batch, would exceed it.  Every proof of the last batch at each
point must equal its known-discrete-log expectation and verify under the real Vk with its witness's own public signal;
otherwise the script exits non-zero.  Prints one JSON line."""
import argparse
import ctypes
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
from gosnark_b200.synthetic import CircuitGroth16, SyntheticCircuit  # noqa: E402
from oracle import ref_py as o  # noqa: E402

G1, G2, R = o.BN.G1, o.BN.G2, o.R


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


def pk_bytes(L, pk):
    v = ctypes.c_size_t(0)
    check(L.b200_pk_device_bytes(pk, ctypes.byref(v)))
    return v.value


def time_ms(run, count, streams, warmup, steps):
    """ms per proof: `run(j, stream)` issues one batch / proof on stream j; one event pair brackets all steps on all
    streams."""
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


def check_proofs(syn, words, wits, pubs, rs, ss):
    """Every proof: its known discrete logs and the real Vk with its own public signal."""
    bad = []
    for p in range(len(wits)):
        w = words[48 * p:48 * p + 48]
        a, c, b = (np.ascontiguousarray(x) for x in (w[:12], w[12:24], w[24:48]))
        ea, eb, ec = syn.expected_dlogs(wits[p], rs[p], ss[p])
        ok = (G1.affine(_unflatten_g1(a)[0]) == G1.affine(G1.mul_scalar(G1.G, ea))
              and G2.affine(_unflatten_g2(b)[0]) == G2.affine(G2.mul_scalar(G2.G, eb))
              and G1.affine(_unflatten_g1(c)[0]) == G1.affine(G1.mul_scalar(G1.G, ec)))
        vk_ok = ctypes.c_int(0)
        pub = ints_to_limbs(pubs[p])
        check(_lib.lib().b200_groth16_verify(ptr(syn.ic), syn.npublic + 1, ptr(syn.alpha1), ptr(syn.beta2), ptr(syn.gamma2),
                                             ptr(syn.delta2), ptr(a), ptr(b), ptr(c), ptr(pub), len(pubs[p]),
                                             ctypes.byref(vk_ok)))
        if not (ok and vk_ok.value):
            bad.append(p)
    return bad


def bench_size(L, logn, ks, args):
    syn = CircuitGroth16(logn)
    pks = []
    try:
        for ctx in range(2):
            check(L.b200_config(_lib.CFG_PK_CONTEXT, ctx))
            pks.append(syn.load_pk())
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))
    h, m = syn.r1cs.handle, syn.m
    kmax = max(ks)
    cs = [SyntheticCircuit(syn.n, seed=0xB47C4 + p) for p in range(kmax)]
    wits, pubs = [c.witness for c in cs], [c.public_signals for c in cs]
    d_w = torch.from_numpy(ints_to_limbs([v for w in wits for v in w]).view(np.int64)).cuda()
    rs = [(syn.r + 7 * p) % R for p in range(kmax)]
    ss = [(syn.s + 11 * p) % R for p in range(kmax)]
    r_l, s_l = ints_to_limbs(rs), ints_to_limbs(ss)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    out = torch.zeros(48 * kmax, dtype=torch.int64, device="cuda")
    outs1 = [torch.zeros(48, dtype=torch.int64, device="cuda") for _ in range(2)]

    def single(c, st):   # proof on stream c on the context-c key
        check(L.b200_groth16_prove_witness_device(pks[c], h, d_w.data_ptr(), m, ptr(r_l[c:c + 1]), ptr(s_l[c:c + 1]),
                                                  outs1[c].data_ptr(), st.cuda_stream))
    res = {"n": syn.n, "m": m, "single_one_at_a_time_ms": time_ms(single, 1, [streams[0]], args.warmup, args.steps),
           "single_two_in_flight_ms": time_ms(single, 1, streams, args.warmup, args.steps)}
    base = pk_bytes(L, pks[0])
    per_proof = None
    points = []
    for k in ks:
        if per_proof is not None and k * per_proof / 2 ** 30 > args.max_gib:
            points.append({"k": k, "skipped": f"scratch estimate {k * per_proof / 2 ** 30:.1f} GiB > --max-gib"})
            continue

        def batch(_, st, k=k):
            check(L.b200_groth16_prove_witness_batch_device(pks[0], h, d_w.data_ptr(), m, k, ptr(r_l), ptr(s_l), out.data_ptr(),
                                                            st.cuda_stream))
        ms = time_ms(batch, k, [streams[0]], args.warmup, args.steps)
        if per_proof is None:
            # the key's scratch of one proof, doubled for the R1CS workspace's batch front end (not counted by the key)
            per_proof = 2 * (pk_bytes(L, pks[0]) - base)
        batch(0, streams[0])
        torch.cuda.synchronize()
        bad = check_proofs(syn, out.cpu().numpy().view(np.uint64), wits[:k], pubs[:k], rs[:k], ss[:k])
        points.append({"k": k, "ms_per_proof": round(ms, 4), "bad_proofs": bad})
    res["points"] = points
    res["pk_device_bytes_after_largest_batch"] = pk_bytes(L, pks[0])
    for pk in pks:
        check(L.b200_pk_free(pk))
    syn.r1cs.free()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--logn", type=int, nargs="+", default=[10, 12, 14, 16])
    ap.add_argument("--k", type=int, nargs="+", default=[1, 2, 4, 8, 16, 32, 64])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--max-gib", type=float, default=40.0)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 1 or min(args.k) < 1:
        ap.error("--steps, --warmup and every k must be >= 1")
    if not torch.cuda.is_available():
        raise SystemExit("batch_prove_bench: no CUDA device (the library has no CPU fallback)")
    _lib.init(0)
    L = _lib.lib()
    sizes = [bench_size(L, logn, sorted(set(args.k)), args) for logn in args.logn]
    name, power = card()
    ok = all(not p.get("bad_proofs") for s in sizes for p in s["points"])
    print(json.dumps({"workload": "batched witness-fed Groth16, CircuitGroth16", "gpu": name, "power_limit": power,
                      "steps": args.steps, "warmup": args.warmup, "sizes": sizes, "ok": ok}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
