"""Reduced window tables (B200_CFG_TABLE_WINDOWS), measured: for SyntheticCircuit(2^logn) and each t in --t, the device
memory of the Groth16 proving key (b200_pk_device_bytes), the key's load time, the time of one proof at a time (median of
--reps after a warm-up) and whether b200_groth16_verify accepts it and rejects a wrong public input; then the time of a
stand-alone G1 MSM of 2^--msm-logn terms per t (b200_msm_device, CUDA events, median of --reps).  t = 0 is the full table.
The key comes from groth16.GenerateTrustedSetupSparse on the device.  --px proves from px (b200_groth16_prove, px from the
sparse front end) instead of from the witness (b200_groth16_prove_witness), for circuits whose witness-fed QAP domains do
not fit next to the key.  Prints one JSON line with the card's name and power limit.

    python tools/table_windows_bench.py --logn 20 --t 0 1 3
    python tools/table_windows_bench.py --logn 24 --t 1 3 --px --reps 1 --msm-logn 0
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gosnark_b200 import _lib, groth16  # noqa: E402
from gosnark_b200._lib import check, ints_to_limbs, lib, ptr  # noqa: E402
from gosnark_b200.bn128 import BaseSet  # noqa: E402
from gosnark_b200.r1csqap import SparseR1CS  # noqa: E402
from gosnark_b200.synthetic import SyntheticCircuit, rand_limbs  # noqa: E402
from oracle import ref_py as o  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


def key_run(setup, sp, w, pub, px, t, reps):
    r, s = 12345, 67890
    t0 = time.perf_counter()
    dpk = setup.load_pk(table_windows=t)
    res = {"t": t, "load_s": round(time.perf_counter() - t0, 3), "pk_device_bytes": dpk.device_bytes()}
    try:
        prove = (lambda: dpk.prove_limbs(w, px, r, s)) if px is not None else (lambda: dpk.prove_witness_limbs(sp, w, r, s))
        proof = prove()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            proof = prove()
            ts.append(time.perf_counter() - t0)
        res["prove_s"] = round(statistics.median(ts), 4) if ts else None
        res["verifies"] = bool(groth16.VerifyProof(setup.Vk, proof, [pub]))
        res["rejects_wrong_public"] = not groth16.VerifyProof(setup.Vk, proof, [(pub + 1) % o.R])
    finally:
        dpk.free()
    return res


def msm_run(logn, t, reps):
    import torch
    n = 1 << logn
    pts = np.zeros((n, 12), dtype=np.uint64)
    k = rand_limbs(n, 7)
    k[:, 3] &= np.uint64((1 << 60) - 1)
    check(lib().b200_g1_mul_batch_bcast(ptr(np.array([1, 0, 0, 0, 2, 0, 0, 0, 1, 0, 0, 0], np.uint64)), ptr(k), n, ptr(pts)))
    bs = BaseSet(1, limbs=pts, table_windows=t)
    try:
        s = rand_limbs(n, 8)
        s[:, 3] &= np.uint64((1 << 60) - 1)
        d_s = torch.from_numpy(s.view(np.int64)).cuda()
        d_out = torch.zeros(16, dtype=torch.int64, device="cuda")
        st = torch.cuda.Stream()
        run = lambda: check(lib().b200_msm_device(bs.handle, d_s.data_ptr(), n, 0, d_out.data_ptr(), st.cuda_stream))
        run()
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            run()
            e1.record(st)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return {"t": t, "msm_ms": round(statistics.median(ts), 3), "bases_device_bytes": bs.device_bytes(),
                "window_bits": bs.info()["window_bits"], "acc_mode": bs.acc_mode()}
    finally:
        bs.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logn", type=int, default=20)
    ap.add_argument("--t", type=int, nargs="+", default=[0, 1, 3])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--px", action="store_true")
    ap.add_argument("--msm-logn", type=int, default=20, help="0: skip the stand-alone MSM")
    a = ap.parse_args()
    _lib.init(0)
    name, power = card()
    out = {"gpu": name, "power_limit": power, "logn": a.logn, "keys": [], "msm": []}
    n = 1 << a.logn
    t0 = time.perf_counter()
    circ = SyntheticCircuit(n)
    sp = SparseR1CS(n, circ.m, circ.csr)
    setup = groth16.GenerateTrustedSetupSparse(sp, circ.npublic)
    out["setup_s"] = round(time.perf_counter() - t0, 3)
    w = ints_to_limbs(circ.witness)
    px = None
    if a.px:
        px = sp.combine_limbs(w, want_abc=False)[3]
        # the px-fed proof needs neither the R1CS nor the interpolation domains and polynomial workspaces that the setup
        # and the front end left cached on the device: start the library afresh so that the keys get the whole card
        sp.free()
        sp = None
        check(lib().b200_shutdown())
        _lib.init(0)
    for t in a.t:
        out["keys"].append(key_run(setup, sp, w, circ.public_signals[0], px, t, a.reps))
        print(json.dumps(out["keys"][-1]), file=sys.stderr, flush=True)
    del setup, px
    if sp is not None:
        sp.free()
    if a.msm_logn:
        for t in a.t:
            out["msm"].append(msm_run(a.msm_logn, t, a.reps))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
