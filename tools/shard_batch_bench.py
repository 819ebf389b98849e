#!/usr/bin/env python3
"""Batched witness-fed Groth16 proving on key shards, every rank of an N-way shard emulated on ONE GPU (development aid;
bench.py is the contract).

CircuitGroth16 for each --logn (a real CRS with known discrete logs, one resident R1CS).  For each N in --worlds the key
is loaded shard by shard (b200_groth16_pk_load_shard, one rank's key at a time).  Each rank's
b200_groth16_prove_witness_batch_partial_device is timed with CUDA events over whole batches for each k in --ks, and the
same rank's single witness-fed proof (b200_groth16_prove_witness_device, its partial record) beside it.  Per (N, n, k)
the line reports the slowest rank's ms per proof in the batch, and that rank's single-proof ms.  With N = 1 the "rank" is
the whole key.  The emulation has no communicator and times no all-gather.  With two or more visible GPUs the line also
has "spmd": a real run over NCCL on every visible GPU (up to 8), one process per GPU, each timing
b200_groth16_prove_witness_batch_device on its shard (all-gather and finalisation included), with the slowest rank's ms
per proof per k; with one GPU it says "not run".  After timing, every rank's records of the largest batch that ran on every rank are finalised and
its first and last proof must equal their known-discrete-log expectations (a k whose scratch does not fit in
device memory is reported as null); otherwise the script exits non-zero.  Prints one JSON line,
with the card's name and power limit read in the same run."""
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
from gosnark_b200.synthetic import CircuitGroth16, SyntheticCircuit  # noqa: E402
from oracle import ref_py as o  # noqa: E402

G1, G2, R = o.BN.G1, o.BN.G2, o.R


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def blindings(k):
    return [((0x1234567 * (p + 3)) << 180 | p) % R for p in range(k)], [((0x7654321 * (p + 5)) << 170 | p) % R for p in range(k)]


def time_ms(run, stream, warmup, steps):
    """ms per call of run() from CUDA events on `stream`, the stream every call enqueues on."""
    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        run()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def emulated(L, syn, world, ks, d_w, warmup, steps):
    """Per rank {k: batch ms per proof (None: the batch did not fit in device memory), "single": single-proof ms}, and
    the finalised proofs of the largest batch that ran on every rank (with their count)."""
    kmax = max(ks)
    rs, ss = blindings(kmax)
    r_l, s_l = ints_to_limbs(rs), ints_to_limbs(ss)
    st = torch.cuda.Stream()
    stream = st.cuda_stream
    per_rank, recs = [], []
    for g in range(world):
        pk = syn.load_pk(g, world)
        rec = torch.zeros(128 * kmax, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()

        def batch(k):
            check(L.b200_groth16_prove_witness_batch_partial_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, k, ptr(r_l),
                                                                    ptr(s_l), rec.data_ptr(), stream))

        def single():
            check(L.b200_groth16_prove_witness_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, ptr(r_l), ptr(s_l),
                                                      rec.data_ptr(), stream))
        times = {"single": time_ms(single, st, warmup, steps)}
        done = 0
        for k in sorted(ks):
            try:
                times[k] = time_ms(lambda: batch(k), st, warmup, steps) / k
                done = k
            except _lib.B200Error as e:
                if "ENOMEM" not in str(e):
                    raise
                times.update({kk: None for kk in ks if kk >= k})
                # scratch grown part-way stays allocated on the key and on the R1CS: start from fresh ones
                check(L.b200_pk_free(pk))
                syn.r1cs.free()
                syn.r1cs = syn.r1cs.__class__(syn.n, syn.m, syn.circuit.csr)
                pk = syn.load_pk(g, world)
                break
        if done:
            batch(done)                 # the records the check below finalises
        torch.cuda.synchronize()
        check(L.b200_pk_free(pk))
        per_rank.append(times)
        recs.append((rec, done))
    kc = min(d for _, d in recs)
    if kc == 0:                         # no batch ran on some rank: nothing to finalise
        return per_rank, None, rs, ss, 0
    parts = torch.cat([r[:128 * kc] for r, _ in recs])
    out = torch.zeros(48 * kc, dtype=torch.int64, device="cuda")
    pk0 = syn.load_pk(0, world)
    torch.cuda.synchronize()
    check(L.b200_groth16_finalize_batch_device(pk0, parts.data_ptr(), world, kc, out.data_ptr(), stream))
    torch.cuda.synchronize()
    check(L.b200_pk_free(pk0))
    return per_rank, out.cpu().numpy().view(np.uint64), rs, ss, kc


def _spmd_worker(rank, world, uid, logn, ks, warmup, steps, ret):
    """One rank of an SPMD run: b200_groth16_prove_witness_batch_device on its shard through the communicator; ms per
    proof from CUDA events on its stream, and whether the first proof of the largest batch is right."""
    try:
        _lib.init(rank)
        torch.cuda.set_device(rank)
        L = _lib.lib()
        n = 1 << logn
        syn = CircuitGroth16(n=n)
        check(L.b200_comm_init(ptr(np.frombuffer(uid, dtype=np.uint8).copy()), rank, world))
        pk = syn.load_pk(rank, world)
        kmax = max(ks)
        wit = SyntheticCircuit(n, seed=0x5EED0).witness
        wl = ints_to_limbs(wit * kmax)
        d_w = torch.from_numpy(wl.reshape(-1).view(np.int64)).cuda()
        out = torch.zeros(48 * kmax, dtype=torch.int64, device="cuda")
        rs, ss = blindings(kmax)
        r_l, s_l = ints_to_limbs(rs), ints_to_limbs(ss)
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        times = {}
        for k in ks:
            times[k] = time_ms(lambda: check(L.b200_groth16_prove_witness_batch_device(
                pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, k, ptr(r_l), ptr(s_l), out.data_ptr(), st.cuda_stream)),
                st, warmup, steps) / k
        w = out.cpu().numpy().view(np.uint64)[:48]
        pa = _unflatten_g1(w[:24])[0]
        ea = syn.expected_dlogs(wit, rs[0], ss[0])[0]
        ok = G1.affine(pa) == G1.affine(G1.mul_scalar(G1.G, ea))
        check(L.b200_pk_free(pk))
        check(L.b200_comm_destroy())
        ret.put((rank, times, ok))
    except Exception as e:   # noqa: BLE001 - reported to the parent
        ret.put((rank, repr(e), False))


def spmd(logn, ks, warmup, steps):
    """Real SPMD over NCCL on every visible GPU (2 .. 8): the slowest rank's ms per proof per k."""
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 8)
    L = _lib.lib()
    uid = np.zeros(128, dtype=np.uint8)
    check(L.b200_comm_unique_id(ptr(uid)))
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_spmd_worker, args=(g, world, uid.tobytes(), logn, ks, warmup, steps, ret)) for g in range(world)]
    for p in procs:
        p.start()
    got = [ret.get(timeout=1800) for _ in range(world)]
    for p in procs:
        p.join(60)
    if any(isinstance(t, str) for _, t, _ in got):
        return {"logn": logn, "world": world, "error": [t for _, t, _ in got if isinstance(t, str)][0]}, False
    return ({"logn": logn, "world": world, "points": [{"k": k, "slowest_rank_ms_per_proof": round(max(t[k] for _, t, _ in got), 4)}
                                                      for k in ks]}, all(ok for _, _, ok in got))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--logn", type=int, nargs="+", default=[16])
    ap.add_argument("--worlds", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 2, 4, 8, 16])
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    _lib.init(0)
    L = _lib.lib()
    name, power = card()
    res = {"tool": "shard_batch_bench", "gpu": name, "power_limit": power, "unit": "ms per proof", "points": []}
    ok = True
    for logn in a.logn:
        n = 1 << logn
        syn = CircuitGroth16(n=n)
        kmax = max(a.ks)
        two = [SyntheticCircuit(n, seed=0x5EED0 + p) for p in range(2)]    # proof p proves witness p % 2
        cs = [two[p % 2] for p in range(kmax)]
        wl = ints_to_limbs([v for c in cs for v in c.witness])
        d_w = torch.from_numpy(wl.reshape(-1).view(np.int64)).cuda()
        torch.cuda.synchronize()
        for world in a.worlds:
            per_rank, raw, rs, ss, kc = emulated(L, syn, world, a.ks, d_w, a.warmup, a.steps)
            for p in (sorted({0, kc - 1}) if kc else []):
                w = raw[48 * p:48 * p + 48]
                pa, pc = _unflatten_g1(w[:24])
                pb = _unflatten_g2(w[24:48])[0]
                ea, eb, ec = syn.expected_dlogs(cs[p].witness, rs[p], ss[p])
                good = (G1.affine(pa) == G1.affine(G1.mul_scalar(G1.G, ea)) and G2.affine(pb) == G2.affine(G2.mul_scalar(G2.G, eb))
                        and G1.affine(pc) == G1.affine(G1.mul_scalar(G1.G, ec)))
                ok = ok and good
            for k in a.ks:
                if any(t[k] is None for t in per_rank):
                    res["points"].append({"logn": logn, "world": world, "k": k, "batch_ms_per_proof": None,
                                          "note": "batch scratch did not fit in device memory on some rank"})
                    continue
                slow = max(range(world), key=lambda g: per_rank[g][k])
                res["points"].append({"logn": logn, "world": world, "k": k, "slowest_rank": slow,
                                      "batch_ms_per_proof": round(per_rank[slow][k], 4),
                                      "single_ms": round(per_rank[slow]["single"], 4),
                                      "slowest_single_ms": round(max(t["single"] for t in per_rank), 4)})
            print(f"# logn {logn} world {world}: " + " ".join(f"k={p['k']}:{p['batch_ms_per_proof']}" for p in res["points"][-len(a.ks):])
                  + f" single(slowest rank) {max(t['single'] for t in per_rank):.3f}", file=sys.stderr, flush=True)
        syn.r1cs.free()
    if torch.cuda.device_count() >= 2:
        res["spmd"] = []
        for logn in a.logn:
            line, good = spmd(logn, a.ks, a.warmup, a.steps)
            res["spmd"].append(line)
            ok = ok and good
    else:
        res["spmd"] = f"not run ({torch.cuda.device_count()} visible GPU)"
    res["proofs_checked"] = ok
    print(json.dumps(res))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
