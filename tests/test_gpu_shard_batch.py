"""GPU: batched witness-fed Groth16 proving on key shards (include/b200snark.h:
b200_groth16_prove_witness_batch_partial_device, b200_groth16_finalize_batch_device, and the batch entries with a
communicator).

Unless a test says otherwise the ranks are emulated on one GPU: every rank's k partial records, concatenated rank-major
as an all-gather of k records per rank leaves them, go through b200_groth16_finalize_batch_device, and each proof must
equal the unsharded batch's proof and the known-discrete-log proof of CircuitGroth16 (a satisfying witness's proof also
verifies under the real Vk; an unsatisfied one's equals the unsharded proof and does not verify)."""
import ctypes
import os

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
G1, G2 = o.BN.G1, o.BN.G2
R = o.R
EINVAL, ERANGE = -3, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


_circuits = {}


def circuit(n):
    from gosnark_b200.synthetic import CircuitGroth16
    if n not in _circuits:
        _circuits[n] = CircuitGroth16(n=n)
    return _circuits[n]


def witnesses(n, k, seed=0):
    """k satisfying witnesses of SyntheticCircuit(n) (ints), their public signals, and which are satisfied: with k >= 3
    witness 1 has one signal off (an unsatisfied witness)."""
    from gosnark_b200.synthetic import SyntheticCircuit
    cs = [SyntheticCircuit(n, seed=0x5BA7C + 977 * seed + p) for p in range(k)]
    wits, pubs = [list(c.witness) for c in cs], [c.public_signals for c in cs]
    sat = [True] * k
    if k >= 3:
        wits[1][n // 2 + 2] = (wits[1][n // 2 + 2] + 1) % R
        sat[1] = False
    return wits, pubs, sat


def blindings(k, seed=0):
    return ([((0x1234567 * (p + 3) + seed) << 180 | p) % R for p in range(k)],
            [((0x7654321 * (p + 5) + seed) << 170 | p) % R for p in range(k)])


def limbs(vals):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs(list(vals))


def _p(a):
    from gosnark_b200._lib import ptr
    return ptr(a)


def to_dev(arr):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


def split(words):
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    pa, pc = _unflatten_g1(words[:24])
    return pa, _unflatten_g2(words[24:48])[0], pc


def affine(p):
    pa, pb, pc = p
    return G1.affine(pa), G2.affine(pb), G1.affine(pc)


def expected(dlogs):
    a, b, c = dlogs
    return G1.affine(G1.mul_scalar(G1.G, a)), G2.affine(G2.mul_scalar(G2.G, b)), G1.affine(G1.mul_scalar(G1.G, c))


def verify_with(syn, proof, public):
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
    from gosnark_b200._lib import check, ints_to_limbs, lib, ptr
    ok = ctypes.c_int(0)
    pa, pb, pc = proof
    pub = ints_to_limbs(public)
    check(lib().b200_groth16_verify(ptr(syn.ic), syn.npublic + 1, ptr(syn.alpha1), ptr(syn.beta2), ptr(syn.gamma2),
                                    ptr(syn.delta2), ptr(_flatten_g1([pa])), ptr(_flatten_g2([pb])), ptr(_flatten_g1([pc])),
                                    ptr(pub), len(public), ctypes.byref(ok)))
    return bool(ok.value)


def with_config(L, fn, ctx=0, acc=0, t=0, weights=None):
    """fn() with the key-load configuration set, restored afterwards."""
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    w_ab, w_g2 = weights or (100, 280)
    try:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, ctx))
        check(L.b200_config(_lib.CFG_ACC_MODE, acc))
        check(L.b200_config(_lib.CFG_TABLE_WINDOWS, t))
        check(L.b200_config(_lib.CFG_SHARD_W_AB, w_ab))
        check(L.b200_config(_lib.CFG_SHARD_W_G2, w_g2))
        return fn()
    finally:
        check(L.b200_config(_lib.CFG_PK_CONTEXT, 0))
        check(L.b200_config(_lib.CFG_ACC_MODE, 0))
        check(L.b200_config(_lib.CFG_TABLE_WINDOWS, 0))
        check(L.b200_config(_lib.CFG_SHARD_W_AB, 100))
        check(L.b200_config(_lib.CFG_SHARD_W_G2, 280))


def shard_info(L, pk):
    from gosnark_b200._lib import check
    info = np.zeros(12, dtype=np.uint64)
    check(L.b200_groth16_shard_info(pk, _p(info)))
    return [int(x) for x in info]


def partial_records(L, pks, r1cs, d_w, m, k, rs, ss, stream=None):
    """Every rank's k records, rank-major (world x k x 1 KB)."""
    import torch
    from gosnark_b200._lib import check
    world = len(pks)
    parts = torch.full((128 * world * k,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()                 # the fill, before other streams write the records
    for g, pk in enumerate(pks):
        check(L.b200_groth16_prove_witness_batch_partial_device(pk, r1cs, d_w.data_ptr(), m, k, _p(limbs(rs)), _p(limbs(ss)),
                                                                parts[128 * k * g:].data_ptr(),
                                                                None if stream is None else stream.cuda_stream))
    return parts


def finalize(L, pk, parts, world, k, stream=None):
    import torch
    from gosnark_b200._lib import check
    d_out = torch.full((48 * k,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    check(L.b200_groth16_finalize_batch_device(pk, parts.data_ptr(), world, k, d_out.data_ptr(),
                                               None if stream is None else stream.cuda_stream))
    torch.cuda.synchronize()
    raw = d_out.cpu().numpy().view(np.uint64)
    return [split(raw[48 * p:48 * p + 48]) for p in range(k)]


def sharded_batch(L, pks, r1cs, d_w, m, rs, ss):
    k = len(rs)
    return finalize(L, pks[0], partial_records(L, pks, r1cs, d_w, m, k, rs, ss), len(pks), k)


def unsharded_batch(L, pk, r1cs, d_w, m, rs, ss):
    import torch
    from gosnark_b200._lib import check
    k = len(rs)
    d_out = torch.full((48 * k,), -1, dtype=torch.int64, device="cuda")
    check(L.b200_groth16_prove_witness_batch_device(pk, r1cs, d_w.data_ptr(), m, k, _p(limbs(rs)), _p(limbs(ss)),
                                                    d_out.data_ptr(), None))
    torch.cuda.synchronize()
    raw = d_out.cpu().numpy().view(np.uint64)
    return [split(raw[48 * p:48 * p + 48]) for p in range(k)]


def load_shards(L, syn, world, **cfg):
    return with_config(L, lambda: [syn.load_pk(g, world) for g in range(world)], **cfg)


def free(L, pks):
    from gosnark_b200._lib import check
    for pk in pks:
        check(L.b200_pk_free(pk))


def check_proofs(syn, got, ref, wits, pubs, sat, rs, ss):
    for p in range(len(got)):
        assert affine(got[p]) == affine(ref[p]), p
        if sat[p]:
            assert affine(got[p]) == expected(syn.expected_dlogs(wits[p], rs[p], ss[p])), p
        assert verify_with(syn, got[p], pubs[p]) == sat[p], p


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("n,world,acc,weights", [
    (1 << 10, 2, 0, None), (1 << 10, 3, 2, (130, 330)), (1 << 10, 8, 1, (85, 275)), (1 << 10, 8, 0, None),
    (1 << 14, 2, 0, None), (1 << 14, 3, 1, None), (1 << 14, 8, 2, None)],
    ids=["1024-w2", "1024-w3-xyzz-weights", "1024-w8-affine-weights", "1024-w8", "16384-w2", "16384-w3-affine", "16384-w8-xyzz"])
def test_shapes(L, n, world, acc, weights):
    syn = circuit(n)
    pk1 = with_config(L, syn.load_pk, acc=acc)
    pks = load_shards(L, syn, world, acc=acc, weights=weights)
    try:
        infos = [shard_info(L, pk) for pk in pks]
        if world == 8 and weights is None:    # a rank without A and B1, and several that need px
            assert any(i[0] == i[1] and i[2] == i[3] for i in infos)
            assert sum(i[8] for i in infos) >= 2
        for k in (1, 3, 8):
            wits, pubs, sat = witnesses(n, k, seed=k)
            rs, ss = blindings(k, seed=k)
            d_w = to_dev(limbs([v for w in wits for v in w]))
            ref = unsharded_batch(L, pk1, syn.r1cs.handle, d_w, syn.m, rs, ss)
            got = sharded_batch(L, pks, syn.r1cs.handle, d_w, syn.m, rs, ss)
            check_proofs(syn, got, ref, wits, pubs, sat, rs, ss)
    finally:
        free(L, pks + [pk1])


def test_world_one_records(L):
    """A world == 1 key's records (the partial entry never combines) finalised with world = 1 give the batch's proofs."""
    n, k = 1 << 10, 4
    syn = circuit(n)
    pk = syn.load_pk()
    try:
        wits, pubs, sat = witnesses(n, k, seed=11)
        rs, ss = blindings(k, seed=11)
        d_w = to_dev(limbs([v for w in wits for v in w]))
        ref = unsharded_batch(L, pk, syn.r1cs.handle, d_w, syn.m, rs, ss)
        got = sharded_batch(L, [pk], syn.r1cs.handle, d_w, syn.m, rs, ss)
        check_proofs(syn, got, ref, wits, pubs, sat, rs, ss)
    finally:
        free(L, [pk])


def _launches(L, fn):
    from gosnark_b200._lib import check
    out = (ctypes.c_double * 8)()
    check(L.b200_profile_read(out))
    fn()
    check(L.b200_profile_read(out))
    return int(out[6])


def pick_window_bits(n):
    """capi.cu's pick_window_bits, restated."""
    best, best_cost = 8, None
    for c in range(8, 19):
        cost = ((255 + c - 1) // c) * n * 10.0 + 2.0 * (1 << (c - 1)) * 14.0 * 4.0
        if best_cost is None or cost < best_cost:
            best, best_cost = c, cost
    return best


def slice_terms(syn, rank, world):
    """Terms of the rank's sets A, B1, B2, C||PTD (0: not held), from the Python mirror of the partition, the distinct
    slices of A / B1 / B2 and whether the rank needs px."""
    from gosnark_b200 import shard
    sr = shard.shard_ranges(syn.m, syn.npublic, syn.n_ptd, rank, world)
    out = []
    for j, st in enumerate(sr["sets"]):
        held = st["lo"] < st["hi"] or st["tail"]
        out.append(st["hi"] - st["lo"] + ((3 if j < 3 else 1) if st["tail"] else 0) if held else 0)
    sorts = {(sr["sets"][j]["lo"], sr["sets"][j]["hi"], sr["sets"][j]["tail"]) for j in range(3) if out[j]}
    return out, sorts, sr["sets"][3]["hi"] > sr["n_c_full"]


def msm_extras(k, c):
    return int(k * (1 << (c - 1)) + 1 > 65536) - int((1 << (c - 1)) + 1 > 65536)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [3, 8])
def test_launch_count_does_not_grow_with_k(L, world):
    """Per rank, from b200_profile_read: the launches of k = 8 are those of k = 1 plus at most b200_msm_device_batch's
    extras of the rank's sets; an 8-way shard has a rank without PowersTauDelta indices (it runs no QAP front end)."""
    n = 1 << 10
    syn = circuit(n)
    pks = load_shards(L, syn, world)
    try:
        wits, _, _ = witnesses(n, 8, seed=5)
        d_w = to_dev(limbs([v for w in wits for v in w]))
        import torch
        from gosnark_b200._lib import check
        d_out = torch.zeros(128 * 8, dtype=torch.int64, device="cuda")
        seen_no_px = False
        for g, pk in enumerate(pks):
            terms, sorts, needs_px = slice_terms(syn, g, world)

            def batch(k):
                rs, ss = blindings(k)
                check(L.b200_groth16_prove_witness_batch_partial_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, k,
                                                                        _p(limbs(rs)), _p(limbs(ss)), d_out.data_ptr(), None))
            for k in (1, 8):
                batch(k)
            base = _launches(L, lambda: batch(1))
            got = _launches(L, lambda: batch(8))
            extras = sum(msm_extras(8, pick_window_bits(t)) for t in terms if t)
            assert base <= got <= base + extras, (g, got, base, extras)
            if not needs_px:
                seen_no_px = True
                assert shard_info(L, pk)[8] == 0
        assert seen_no_px or world < 8
    finally:
        free(L, pks)


@pytest.mark.timeout(900)
def test_reduced_tables_and_two_contexts(L):
    """Shards with one stored window row (B200_CFG_TABLE_WINDOWS = 1) give the same proofs; shards of prove contexts 0
    and 1 batch on two streams at once and give the same proofs."""
    import torch
    n, world, k = 1 << 10, 3, 3
    syn = circuit(n)
    pk1 = syn.load_pk()
    full = load_shards(L, syn, world)
    reduced = load_shards(L, syn, world, t=1)
    ctx1 = load_shards(L, syn, world, ctx=1)
    try:
        wits, pubs, sat = witnesses(n, k, seed=21)
        rs, ss = blindings(k, seed=21)
        d_w = to_dev(limbs([v for w in wits for v in w]))
        ref = unsharded_batch(L, pk1, syn.r1cs.handle, d_w, syn.m, rs, ss)
        check_proofs(syn, sharded_batch(L, reduced, syn.r1cs.handle, d_w, syn.m, rs, ss), ref, wits, pubs, sat, rs, ss)
        s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
        rs2, ss2 = blindings(k, seed=22)
        ref2 = unsharded_batch(L, pk1, syn.r1cs.handle, d_w, syn.m, rs2, ss2)
        p0 = partial_records(L, full, syn.r1cs.handle, d_w, syn.m, k, rs, ss, s0)
        p1 = partial_records(L, ctx1, syn.r1cs.handle, d_w, syn.m, k, rs2, ss2, s1)
        got0 = finalize(L, full[0], p0, world, k, s0)
        got1 = finalize(L, ctx1[0], p1, world, k, s1)
        check_proofs(syn, got0, ref, wits, pubs, sat, rs, ss)
        check_proofs(syn, got1, ref2, wits, pubs, sat, rs2, ss2)
    finally:
        free(L, full + reduced + ctx1 + [pk1])


@pytest.mark.timeout(900)
def test_scratch_regrowth(L):
    """A larger k after a smaller one grows every rank's scratch (b200_pk_device_bytes grows) and gives the right proofs."""
    from gosnark_b200 import _lib
    n, world = 1 << 10, 3
    syn = circuit(n)
    pk1 = syn.load_pk()
    pks = load_shards(L, syn, world)
    try:
        before = None
        for k in (2, 6):
            wits, pubs, sat = witnesses(n, k, seed=30 + k)
            rs, ss = blindings(k, seed=30 + k)
            d_w = to_dev(limbs([v for w in wits for v in w]))
            ref = unsharded_batch(L, pk1, syn.r1cs.handle, d_w, syn.m, rs, ss)
            check_proofs(syn, sharded_batch(L, pks, syn.r1cs.handle, d_w, syn.m, rs, ss), ref, wits, pubs, sat, rs, ss)
            now = [_lib.pk_device_bytes(pk) for pk in pks]
            if before is not None:
                assert all(b > a for a, b in zip(before, now)), (before, now)
            before = now
    finally:
        free(L, pks + [pk1])


@pytest.mark.timeout(900)
def test_errors(L):
    """Every documented code of the partial and finalize entries.  A batch too large for the largest rank's part is
    refused by every rank's key, also by a rank whose own sets would fit.  The batch entries still refuse a sharded key
    without a communicator."""
    import torch
    from gosnark_b200._lib import check
    n, world = 1 << 10, 8
    syn = circuit(n)
    pks = load_shards(L, syn, world)
    m, h = syn.m, syn.r1cs.handle
    try:
        d_w = to_dev(limbs([v for v in witnesses(n, 1)[0][0]] * 2))
        d_out = torch.zeros(128 * 2 * world, dtype=torch.int64, device="cuda")
        rs, ss = blindings(2)
        r_l, s_l = limbs(rs), limbs(ss)
        part = L.b200_groth16_prove_witness_batch_partial_device
        assert part(pks[0], h, d_w.data_ptr(), m, 0, _p(r_l), _p(s_l), d_out.data_ptr(), None) == EINVAL
        assert part(0xdead, h, d_w.data_ptr(), m, 2, _p(r_l), _p(s_l), d_out.data_ptr(), None) == EINVAL
        assert part(pks[0], 0xdead, d_w.data_ptr(), m, 2, _p(r_l), _p(s_l), d_out.data_ptr(), None) == EINVAL
        assert part(pks[0], h, None, m, 2, _p(r_l), _p(s_l), d_out.data_ptr(), None) == EINVAL
        assert part(pks[0], h, d_w.data_ptr(), m, 2, None, _p(s_l), d_out.data_ptr(), None) == EINVAL
        assert part(pks[0], h, d_w.data_ptr(), m, 2, _p(r_l), _p(s_l), None, None) == EINVAL
        assert part(pks[0], h, d_w.data_ptr(), m - 1, 2, _p(r_l), _p(s_l), d_out.data_ptr(), None) == EINVAL
        assert part(pks[0], h, d_w.data_ptr(), m, 2, _p(limbs([rs[0], R])), _p(s_l), d_out.data_ptr(), None) == ERANGE
        assert part(pks[0], h, d_w.data_ptr(), m, 2, _p(r_l), _p(limbs([R + 1, ss[1]])), d_out.data_ptr(), None) == ERANGE
        # too large: k * nwin * terms reaches 2^31 on the largest part; the rank with the smallest part would fit
        parts = [slice_terms(syn, g, world)[0] for g in range(world)]
        entries = [max(((255 + c - 1) // c) * t for t in ts if t for c in [pick_window_bits(t)]) for ts in parts]
        k_big = (1 << 31) // max(entries) + 1
        assert k_big * min(entries) < (1 << 31)
        big_r, big_s = limbs([1] * k_big), limbs([2] * k_big)
        for pk in pks:
            assert part(pk, h, d_w.data_ptr(), m, k_big, _p(big_r), _p(big_s), d_out.data_ptr(), None) == EINVAL
        # the batch entries without a communicator
        pa, pb, pc = np.zeros(24, np.uint64), np.zeros(48, np.uint64), np.zeros(24, np.uint64)
        wl = limbs([v for v in witnesses(n, 1)[0][0]] * 2)
        assert L.b200_groth16_prove_witness_batch(pks[1], h, _p(wl), m, 2, _p(r_l), _p(s_l), _p(pa), _p(pb), _p(pc)) == EINVAL
        assert L.b200_groth16_prove_witness_batch_device(pks[1], h, d_w.data_ptr(), m, 2, _p(r_l), _p(s_l), d_out.data_ptr(),
                                                         None) == EINVAL
        fin = L.b200_groth16_finalize_batch_device
        assert fin(0xdead, d_out.data_ptr(), world, 2, d_out.data_ptr(), None) == EINVAL
        assert fin(pks[0], None, world, 2, d_out.data_ptr(), None) == EINVAL
        assert fin(pks[0], d_out.data_ptr(), world, 2, None, None) == EINVAL
        assert fin(pks[0], d_out.data_ptr(), 0, 2, d_out.data_ptr(), None) == EINVAL
        assert fin(pks[0], d_out.data_ptr(), world, 0, d_out.data_ptr(), None) == EINVAL
        assert fin(pks[0], d_out.data_ptr(), world, 1 << 32, d_out.data_ptr(), None) == EINVAL
        # the keys still prove
        wits, pubs, sat = witnesses(n, 2, seed=40)
        rs, ss = blindings(2, seed=40)
        d_w = to_dev(limbs([v for w in wits for v in w]))
        got = sharded_batch(L, pks, h, d_w, m, rs, ss)
        for p in range(2):
            assert affine(got[p]) == expected(syn.expected_dlogs(wits[p], rs[p], ss[p])), p
    finally:
        free(L, pks)


def _comm_worker(rank, world, uid, n, k, ret):
    import sys
    sys.path.insert(0, ROOT)
    import torch
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check, ptr
    from gosnark_b200.synthetic import CircuitGroth16
    try:
        _lib.init(rank)
        L = _lib.lib()
        syn = CircuitGroth16(n=n)
        pk = syn.load_pk(rank, world)
        check(L.b200_comm_init(ptr(np.frombuffer(uid, dtype=np.uint8).copy()), rank, world))
        wits, _, _ = witnesses(n, k, seed=50)
        rs, ss = blindings(k, seed=50)
        wl = limbs([v for w in wits for v in w])
        pa, pb, pc = np.zeros(12 * k, np.uint64), np.zeros(24 * k, np.uint64), np.zeros(12 * k, np.uint64)
        check(L.b200_groth16_prove_witness_batch(pk, syn.r1cs.handle, ptr(wl), syn.m, k, ptr(limbs(rs)), ptr(limbs(ss)),
                                                 ptr(pa), ptr(pb), ptr(pc)))
        torch.cuda.set_device(rank)
        d_w = torch.from_numpy(wl.reshape(-1).view(np.int64)).cuda()
        d_out = torch.zeros(48 * k, dtype=torch.int64, device="cuda")
        check(L.b200_groth16_prove_witness_batch_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, k, ptr(limbs(rs)),
                                                        ptr(limbs(ss)), d_out.data_ptr(), None))
        torch.cuda.synchronize()
        raw = d_out.cpu().numpy().view(np.uint64)
        ok = True
        for p in range(k):
            want = expected(syn.expected_dlogs(wits[p], rs[p], ss[p]))
            host = split(np.concatenate([pa[12 * p:12 * p + 12], pc[12 * p:12 * p + 12], pb[24 * p:24 * p + 24]]))
            ok = ok and affine(host) == want and affine(split(raw[48 * p:48 * p + 48])) == want
        ret.put((rank, ok))
        check(L.b200_comm_destroy())
    except Exception as e:   # noqa: BLE001 - reported to the parent
        ret.put((rank, repr(e)))


@pytest.mark.timeout(900)
def test_batch_entries_with_communicator(L):
    """SPMD over a real NCCL communicator, one process per GPU: the host and device batch entries on sharded keys return
    all k proofs on every rank.  Needs at least two visible GPUs."""
    import torch
    import torch.multiprocessing as mp
    from gosnark_b200._lib import check, ptr
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs at least two GPUs")
    uid = np.zeros(128, dtype=np.uint8)
    check(L.b200_comm_unique_id(ptr(uid)))
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_comm_worker, args=(rk, world, uid.tobytes(), 1 << 10, 3, ret)) for rk in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
    got = dict(ret.get(timeout=5) for _ in range(world))
    assert all(v is True for v in got.values()), got
    assert all(p.exitcode == 0 for p in procs)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [2, 3, 8])
def test_real_setup_shards_verify(L, world):
    """A key from groth16.GenerateTrustedSetupSparse on CircuitGroth16's R1CS, loaded as `world` shards: every proof of a
    sharded batch equals the unsharded key's batch proof and verifies under the setup's own Vk (b200_groth16_verify);
    the unsatisfied witness's proof is refused."""
    from gosnark_b200 import groth16
    n, k = (1 << 12) + 2, 4
    syn = circuit(n)
    new = groth16.GenerateTrustedSetupSparse(syn.r1cs, syn.npublic, toxic=syn.toxic)
    single = new.load_pk()
    shards = [new.load_pk(rank=g, world=world) for g in range(world)]
    try:
        wits, pubs, sat = witnesses(n, k, seed=60 + world)
        rs, ss = blindings(k, seed=60 + world)
        d_w = to_dev(limbs([v for w in wits for v in w]))
        ref = unsharded_batch(L, single.handle, syn.r1cs.handle, d_w, syn.m, rs, ss)
        got = sharded_batch(L, [pk.handle for pk in shards], syn.r1cs.handle, d_w, syn.m, rs, ss)
        for p in range(k):
            assert affine(got[p]) == affine(ref[p]), p
            pa, pb, pc = got[p]
            assert groth16.VerifyProof(new.Vk, {"PiA": pa, "PiB": pb, "PiC": pc}, pubs[p]) == sat[p], p
    finally:
        for pk in [single] + shards:
            pk.free()


# ---- Pinocchio -----------------------------------------------------------------------------------------------------------
PIN_ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


def pin_split(words):
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    words = np.asarray(words, dtype=np.uint64)
    return list(_unflatten_g1(words[:84])) + [_unflatten_g2(words[84:108])[0]]


def pin_affine(p):
    return [G1.affine(q) for q in p[:7]] + [G2.affine(p[7])]


def pin_unsharded(L, pk, r1cs, d_w, m, k):
    import torch
    from gosnark_b200._lib import check
    d_out = torch.full((108 * k,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    check(L.b200_pinocchio_prove_witness_batch_device(pk, r1cs, d_w.data_ptr(), m, k, d_out.data_ptr(), None))
    torch.cuda.synchronize()
    raw = d_out.cpu().numpy().view(np.uint64)
    return [pin_split(raw[108 * p:108 * p + 108]) for p in range(k)]


def pin_sharded(L, pks, r1cs, d_w, m, k):
    """Every rank's k records (rank-major) through b200_pinocchio_finalize_records_batch_device."""
    import torch
    from gosnark_b200._lib import check
    world = len(pks)
    recs = torch.full((256 * world * k,), -1, dtype=torch.int64, device="cuda")
    d_out = torch.full((108 * k,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for g, pk in enumerate(pks):
        check(L.b200_pinocchio_prove_witness_batch_record_device(pk, r1cs, d_w.data_ptr(), m, k, recs[256 * k * g:].data_ptr(),
                                                                 None))
    check(L.b200_pinocchio_finalize_records_batch_device(recs.data_ptr(), world, k, d_out.data_ptr(), None))
    torch.cuda.synchronize()
    raw = d_out.cpu().numpy().view(np.uint64)
    return [pin_split(raw[108 * p:108 * p + 108]) for p in range(k)]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("world", [2, 3, 8])
def test_pinocchio_shards_equal_unsharded(L, world):
    """CircuitPinocchio at 2^10: each rank runs only the sets it owns; the finalised records equal the unsharded batch and,
    for satisfying witnesses, the known-discrete-log proof.  Every rank's launches at k = 8 equal those at k = 1 (no
    batched-MSM extras at this size)."""
    from gosnark_b200._lib import check
    from gosnark_b200.synthetic import CircuitPinocchio
    n = 1 << 10
    syn = CircuitPinocchio(n)
    pk1 = syn.load_pk()
    pks = [syn.load_pk(g, world) for g in range(world)]
    try:
        for k in (1, 3, 8):
            wits, pubs, sat = witnesses(n, k, seed=70 + k)
            d_w = to_dev(limbs([v for w in wits for v in w]))
            ref = pin_unsharded(L, pk1, syn.r1cs.handle, d_w, syn.m, k)
            got = pin_sharded(L, pks, syn.r1cs.handle, d_w, syn.m, k)
            for p in range(k):
                assert pin_affine(got[p]) == pin_affine(ref[p]), p
                if sat[p]:
                    want = syn.expected_dlogs(wits[p])
                    exp = [G1.affine(G1.mul_scalar(G1.G, want[kk])) for kk in PIN_ORDER] + [G2.affine(G2.mul_scalar(G2.G, want["PiB"]))]
                    assert pin_affine(got[p]) == exp, p
        import torch
        d_w = to_dev(limbs([v for w in witnesses(n, 8, seed=79)[0] for v in w]))
        rec = torch.zeros(256 * 8, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        for pk in pks:
            def batch(k):
                check(L.b200_pinocchio_prove_witness_batch_record_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, k,
                                                                         rec.data_ptr(), None))
            batch(8)
            c1, c8 = _launches(L, lambda: batch(1)), _launches(L, lambda: batch(8))
            assert c1 == c8, (c1, c8)
    finally:
        free(L, pks + [pk1])


@pytest.mark.parametrize("name", ["x3x5", "chain21"])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_pinocchio_go_binary_circuits(L, golden_dir, name, world):
    """The Go binary's circuits on sharded keys: a batch of the golden witness twice gives the Go binary's proof."""
    import json
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2, reduce_scalar
    from gosnark_b200.r1csqap import SparseR1CS
    with open(os.path.join(golden_dir, f"gobin_{name}.json")) as f:
        g = json.load(f)
    cc = g["compiledcircuit"]
    a, b, c = cc["R1CS"]["A"], cc["R1CS"]["B"], cc["R1CS"]["C"]
    n, m, npub = len(a), len(a[0]), cc["NPublic"]
    sp = SparseR1CS(n, m, (a, b, c))
    st = g["pinocchio_setup"]
    t3 = tuple
    arr = {k: _flatten_g1([t3(p) for p in st["Pk"][k][:m]]) for k in ("A", "Ap", "Bp", "C", "Cp", "Kp")}
    b2 = _flatten_g2([tuple(tuple(c_) for c_ in p) for p in st["Pk"]["B"][:m]])
    g1t = _flatten_g1([t3(p) for p in st["G1T"]])
    z = ints_to_limbs([int(x) % R for x in st["Pk"]["Z"]])
    handles = []
    try:
        for rk in range(world):
            h = _lib._h(0)
            check(L.b200_pinocchio_pk_load_shard(ptr(arr["A"]), ptr(arr["Ap"]), ptr(b2), ptr(arr["Bp"]), ptr(arr["C"]),
                                                 ptr(arr["Cp"]), ptr(arr["Kp"]), m, ptr(g1t), len(st["G1T"]), ptr(z),
                                                 len(st["Pk"]["Z"]), npub, 0, rk, world, h))
            handles.append(h.value)
        w = [reduce_scalar(x) for x in g["witness"]]
        d_w = to_dev(limbs(w + w))
        got = pin_sharded(L, handles, sp.handle, d_w, m, 2)
        ref = g["pinocchio_proofs"]
        for p in range(2):
            for i, kk in enumerate(("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")):
                assert G1.affine(got[p][i]) == G1.affine(tuple(ref[kk])), (kk, p)
            assert G2.affine(got[p][7]) == G2.affine(tuple(tuple(c_) for c_ in ref["PiB"])), p
        # the batch entries still refuse a sharded key without a communicator
        g1o, pbo = np.zeros(84 * 2, np.uint64), np.zeros(48, np.uint64)
        assert L.b200_pinocchio_prove_witness_batch(handles[0], sp.handle, ptr(limbs(w + w)), m, 2, ptr(g1o), ptr(pbo)) == EINVAL
    finally:
        free(L, handles)
        sp.free()
