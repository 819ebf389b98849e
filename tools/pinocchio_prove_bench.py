#!/usr/bin/env python3
"""Pinocchio proving timed on one GPU (development aid; bench.py is the contract).

CircuitPinocchio(2^logn) for each --logn: a real key and Vk with known discrete logs, one resident R1CS.  ms per proof for
  - b200_pinocchio_prove (px-fed, host pointers: the witness and px cross PCIe, and the call waits), host clock around
    calls that end in a wait;
  - b200_pinocchio_prove_witness_device one at a time and with two in flight (a second key on prove context 1), CUDA
    events over all steps;
  - b200_pinocchio_prove_witness_batch_device for each k over k distinct satisfying witnesses, CUDA events over whole
    batches.
Every figure is the median of --repeats timed windows of --steps steps each, with the fastest and slowest window beside it
(`spread`).  Beside them the key's b200_pk_device_bytes after the largest batch, the window bits and accumulation kernel the
library picks for a base set of the key's m points (they decide the batch scratch: the batched-affine tree keeps node
buffers per slice, XYZZ does not), and the card's name and power limit as read.
--max-gib skips the (n, k) points whose batch scratch, extrapolated from the k = 1 batch, would exceed it.  Every proof of
the last batch at each point must equal its known-discrete-log expectation and verify under the real Vk with its
witness's own public signal; otherwise the script exits non-zero.  Prints one JSON line."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from batch_prove_bench import card, pk_bytes, time_ms  # noqa: E402
from gosnark_b200 import _lib  # noqa: E402
from gosnark_b200._lib import check, ints_to_limbs, ptr  # noqa: E402
from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2  # noqa: E402
from gosnark_b200.synthetic import CircuitPinocchio, SyntheticCircuit  # noqa: E402
from oracle import ref_py as o  # noqa: E402

G1, G2 = o.BN.G1, o.BN.G2
ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


def spread(measure, repeats):
    """Median of `repeats` measurements, and the fastest and slowest of them."""
    v = sorted(measure() for _ in range(repeats))
    return round(v[len(v) // 2], 4), [round(v[0], 4), round(v[-1], 4)]


def set_shape(L, pts):
    """Window bits and accumulation kernel of a G1 base set over `pts`, as the library chooses them for a key's set."""
    h, c, mode = _lib._h(0), ctypes.c_int(0), ctypes.c_int(0)
    check(L.b200_g1_bases_load(ptr(pts), pts.shape[0], 0, ctypes.byref(h)))
    check(L.b200_bases_info(h, None, None, ctypes.byref(c), None))
    check(L.b200_bases_acc_mode(h, ctypes.byref(mode)))
    check(L.b200_bases_free(h))
    return {"window_bits": c.value, "accumulation": "batched affine" if mode.value == 1 else "xyzz"}


def check_proofs(syn, words, wits, pubs):
    """Every proof: its known discrete logs and the real Vk with its own public signal."""
    bad = []
    for p in range(len(wits)):
        w = np.ascontiguousarray(words[108 * p:108 * p + 108])
        proof = dict(zip(ORDER, _unflatten_g1(w[:84])))
        proof["PiB"] = _unflatten_g2(w[84:])[0]
        d = syn.expected_dlogs(wits[p])
        ok = (all(G1.affine(proof[k]) == G1.affine(G1.mul_scalar(G1.G, d[k])) for k in ORDER)
              and G2.affine(proof["PiB"]) == G2.affine(G2.mul_scalar(G2.G, d["PiB"])))
        if not (ok and syn.verify(proof, pubs[p])):
            bad.append(p)
    return bad


def bench_size(L, logn, ks, args):
    syn = CircuitPinocchio(1 << logn)
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
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    out = torch.zeros(108 * kmax, dtype=torch.int64, device="cuda")
    outs1 = [torch.zeros(108, dtype=torch.int64, device="cuda") for _ in range(2)]
    g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)

    def px_fed():
        check(L.b200_pinocchio_prove(pks[0], ptr(syn.w), m, ptr(syn.px), syn.px.shape[0], ptr(g1), ptr(pb)))
    for _ in range(args.warmup):
        px_fed()

    def px_window():
        t0 = time.perf_counter()
        for _ in range(args.steps):
            px_fed()                  # each call ends in a wait for its proof
        return (time.perf_counter() - t0) * 1e3 / args.steps

    def single(c, st):   # proof on stream c on the context-c key
        check(L.b200_pinocchio_prove_witness_device(pks[c], h, d_w.data_ptr(), m, outs1[c].data_ptr(), st.cuda_stream))
    res = {"n": syn.n, "m": m, "set_of_m_points": set_shape(L, syn.pk["C"])}
    for name, measure in (("px_fed_host_ms", px_window),
                          ("single_one_at_a_time_ms", lambda: time_ms(single, 1, [streams[0]], args.warmup, args.steps)),
                          ("single_two_in_flight_ms", lambda: time_ms(single, 1, streams, args.warmup, args.steps))):
        res[name], res[name.replace("_ms", "_spread")] = spread(measure, args.repeats)
    base = pk_bytes(L, pks[0])
    per_proof = None
    points = []
    for k in ks:
        if per_proof is not None and k * per_proof / 2 ** 30 > args.max_gib:
            points.append({"k": k, "skipped": f"scratch estimate {k * per_proof / 2 ** 30:.1f} GiB > --max-gib"})
            continue

        def batch(_, st, k=k):
            check(L.b200_pinocchio_prove_witness_batch_device(pks[0], h, d_w.data_ptr(), m, k, out.data_ptr(), st.cuda_stream))
        ms, sp = spread(lambda: time_ms(batch, k, [streams[0]], args.warmup, args.steps), args.repeats)
        if per_proof is None:
            # the key's scratch of one proof, doubled for the R1CS workspace's batch front end (not counted by the key)
            per_proof = 2 * (pk_bytes(L, pks[0]) - base)
        batch(0, streams[0])
        torch.cuda.synchronize()
        bad = check_proofs(syn, out.cpu().numpy().view(np.uint64), wits[:k], pubs[:k])
        points.append({"k": k, "ms_per_proof": ms, "spread": sp, "bad_proofs": bad})
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-gib", type=float, default=40.0)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 1 or args.repeats < 1 or min(args.k) < 1:
        ap.error("--steps, --warmup, --repeats and every k must be >= 1")
    if not torch.cuda.is_available():
        raise SystemExit("pinocchio_prove_bench: no CUDA device (the library has no CPU fallback)")
    _lib.init(0)
    L = _lib.lib()
    sizes = [bench_size(L, logn, sorted(set(args.k)), args) for logn in args.logn]
    name, power = card()
    ok = all(not p.get("bad_proofs") for s in sizes for p in s["points"])
    print(json.dumps({"workload": "Pinocchio: px-fed, witness-fed and batched, CircuitPinocchio", "gpu": name,
                      "power_limit": power, "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
                      "sizes": sizes, "ok": ok}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
