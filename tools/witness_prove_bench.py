#!/usr/bin/env python3
"""Witness-fed Groth16 proving timed from device memory (development aid; bench.py is the contract).

CircuitGroth16(logn): a real CRS with known discrete logs.  Two proving keys, on prove contexts 0 and 1, share one
resident R1CS.  Four figures, ms per proof from CUDA events: b200_groth16_prove_witness_device one at a time and with
two proofs in flight (proof i on context i mod 2, on stream i mod 2), and the same two for b200_groth16_prove_device fed
the host-computed px.  The last witness-fed proof of each context must equal its known-discrete-log expectation and
verify under the real Vk; otherwise the script exits non-zero.  Prints one JSON line."""
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
from gosnark_b200.synthetic import CircuitGroth16  # noqa: E402
from oracle import ref_py as o  # noqa: E402


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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--logn", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be >= 1 and --warmup >= 0")
    if not torch.cuda.is_available():
        raise SystemExit("witness_prove_bench: no CUDA device (the library has no CPU fallback)")
    _lib.init(0)
    L = _lib.lib()
    syn = CircuitGroth16(args.logn)
    pks = []
    try:
        for k in range(2):
            check(L.b200_config(_lib.CFG_PK_CONTEXT, k))
            pks.append(syn.load_pk())
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))
    h = syn.r1cs.handle
    d_w = torch.from_numpy(syn.w.view(np.int64)).cuda()
    d_px = torch.from_numpy(syn.px.view(np.int64)).cuda()
    npx = syn.px.shape[0]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = [torch.zeros(48, dtype=torch.int64, device="cuda") for _ in range(2)]
    rs = [((syn.r + 7 * k) % o.R, (syn.s + 11 * k) % o.R) for k in range(2)]
    rs_l = [(ints_to_limbs([r]), ints_to_limbs([s])) for r, s in rs]
    torch.cuda.synchronize()

    def witness(k, st):
        check(L.b200_groth16_prove_witness_device(pks[k], h, d_w.data_ptr(), syn.m, ptr(rs_l[k][0]), ptr(rs_l[k][1]),
                                                  outs[k].data_ptr(), st.cuda_stream))

    def device_px(k, st):
        check(L.b200_groth16_prove_device(pks[k], d_w.data_ptr(), syn.m, d_px.data_ptr(), npx, ptr(rs_l[k][0]),
                                          ptr(rs_l[k][1]), outs[k].data_ptr(), st.cuda_stream))

    def ms_per_proof(prove, in_flight):
        """Proof i on the key of context i mod in_flight, on stream i mod in_flight; one event pair brackets all."""
        def run(count):
            for i in range(count):
                k = i % in_flight
                prove(k, streams[k])
        run(args.warmup * in_flight)
        torch.cuda.synchronize()
        e0, e1, e_side = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record(streams[0])
        streams[1].wait_event(e0)
        n = args.steps * in_flight
        run(n)
        e_side.record(streams[1])
        streams[0].wait_event(e_side)
        e1.record(streams[0])
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    res = {
        "witness_one_at_a_time_ms": ms_per_proof(witness, 1),
        "witness_two_in_flight_ms": ms_per_proof(witness, 2),
        "px_one_at_a_time_ms": ms_per_proof(device_px, 1),
        "px_two_in_flight_ms": ms_per_proof(device_px, 2),
    }
    # the last witness-fed proof of each context: known discrete logs and the real Vk
    for k in range(2):
        witness(k, streams[k])
    torch.cuda.synchronize()
    checks = {}
    for k in range(2):
        words = outs[k].cpu().numpy().view(np.uint64)
        a, c = (np.ascontiguousarray(x) for x in (words[:12], words[12:24]))
        b = np.ascontiguousarray(words[24:48])
        ea, eb, ec = syn.expected_dlogs(r=rs[k][0], s=rs[k][1])
        G1, G2 = o.BN.G1, o.BN.G2
        dlogs_ok = (G1.affine(_unflatten_g1(a)[0]) == G1.affine(G1.mul_scalar(G1.G, ea))
                    and G2.affine(_unflatten_g2(b)[0]) == G2.affine(G2.mul_scalar(G2.G, eb))
                    and G1.affine(_unflatten_g1(c)[0]) == G1.affine(G1.mul_scalar(G1.G, ec)))
        checks[f"context{k}"] = {"known_dlogs": bool(dlogs_ok), "verifies": bool(syn.verify(a, b, c))}
    name, power = card()
    ok = all(v for c in checks.values() for v in c.values())
    print(json.dumps({"workload": f"witness-fed Groth16, CircuitGroth16 n = 2^{args.logn}", "n": syn.n, "m": syn.m,
                      "steps": args.steps, "warmup": args.warmup, "gpu": name, "power_limit": power,
                      **{k: round(v, 3) for k, v in res.items()}, "checks": checks, "ok": ok}))
    for pk in pks:
        check(L.b200_pk_free(pk))
    syn.r1cs.free()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
