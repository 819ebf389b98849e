"""GPU: base sets and proving keys with reduced window tables (B200_CFG_TABLE_WINDOWS = t < nwin).

A reduced set stores 2^(c*j) * P_i for j < t only; window w reads row w mod t and feeds the buckets of group w / t, and
the tail recombines the groups with doublings.  Every expected value comes from known discrete logs (one CPU scalar
multiplication by sum s_i k_i mod r, test_gpu_msm_adversarial's helpers); no GPU output feeds an expectation.
  - MSMs (b200_g1_msm / b200_g2_msm / b200_msm_device) at G1 2^14, 2^20 and G2 2^11, 2^18 for t in {1, 2, 3, 7, nwin - 1},
    under both accumulation kernels, on random and adversarial scalar families;
  - Groth16 through all four prove entry points and Pinocchio at 2^12 + 2 and 2^16 constraints with t = 1 and 3, sharded
    Groth16 keys on 2 and 3 ranks, and two prove contexts in flight;
  - memory (b200_pk_device_bytes, b200_bases_device_bytes), the launch count of the grouped tail, and the option's
    argument checks."""
import ctypes

import numpy as np
import pytest

import test_gpu_msm_adversarial as adv
import test_gpu_prove_degenerate as deg
from oracle import ref_py as o

pytestmark = pytest.mark.gpu

R = o.R
G1, G2 = o.BN.G1, o.BN.G2
EINVAL = -3
CFG_TABLE_WINDOWS = 14


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


def table_ts(c):
    nwin = adv.n_windows(c)
    return sorted({1, 2, 3, 7, nwin - 1})


def load(g, pool, n, mode, t):
    from gosnark_b200 import bn128
    pts = np.ascontiguousarray(pool[np.arange(n) % pool.shape[0]])
    return bn128.BaseSet(g, limbs=pts, acc_mode=mode, table_windows=t)


def msm_device(L, bs, s):
    """b200_msm_device on a side stream, summed by b200_g*_sum_partials: the set's output for scalar limbs s."""
    import torch
    from gosnark_b200._lib import check, ptr
    d_s = torch.from_numpy(np.ascontiguousarray(s).view(np.int64)).cuda()
    d_rec = torch.zeros(adv.REC_WORDS[bs.group], dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    check(L.b200_msm_device(bs.handle, d_s.data_ptr(), s.shape[0], 0, d_rec.data_ptr(), side.cuda_stream))
    side.synchronize()
    out = np.zeros(12 if bs.group == 1 else 24, dtype=np.uint64)
    fn = L.b200_g1_sum_partials if bs.group == 1 else L.b200_g2_sum_partials
    check(fn(d_rec.data_ptr(), 1, ptr(out), None))
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    return _unflatten_g1(out)[0] if bs.group == 1 else _unflatten_g2(out)[0]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("g,logn", adv.SHAPES, ids=[f"G{g}-n{1 << lg}" for g, lg in adv.SHAPES])
def test_reduced_table_msm_known_dlogs(L, g, logn, mode):
    """For every t: the set stores t rows, takes the accumulation kernel the rules give, and every scalar family returns
    the known-discrete-log point through the host and the device entry points."""
    n = 1 << logn
    c = adv.pick_window_bits(n)
    ks, pool = adv.base_pool(g, "pm-pairs", c, seed=77 * g + logn)
    fam = adv.scalar_families(n, c, seed=3 * logn + g)
    rng = np.random.default_rng(logn)
    fam["random"] = adv.full_width(n, rng)
    exp = {name: adv.expect_out(g, adv.dlog(ks, s)) for name, s in fam.items()}
    for t in table_ts(c):
        bs = load(g, pool, n, mode, t)
        try:
            assert bs.table_windows() == t and bs.info()["n_windows"] == adv.n_windows(c)
            groups = -(-adv.n_windows(c) // t)
            affine_ok = adv.n_windows(c) * n // (groups << (c - 1)) >= 16
            assert bs.acc_mode() == (1 if mode == 1 and affine_ok else 2), t
            for name, s in fam.items():
                assert bs.msm(limbs=s) == exp[name], (t, name)
            assert msm_device(L, bs, fam["random"]) == exp["random"], t
            assert msm_device(L, bs, fam["digits"]) == exp["digits"], t
        finally:
            bs.free()


def test_auto_mode_takes_xyzz_on_reduced_tables(L):
    """B200_CFG_ACC_MODE 0 gives a set with t < nwin the XYZZ kernel and a full set the batched-affine one."""
    n = 1 << 20                                             # populated enough for the batched-affine kernel with full tables
    ks, pool = adv.base_pool(1, "pm-pairs", adv.pick_window_bits(n), seed=5)
    full, red = load(1, pool, n, 0, 0), load(1, pool, n, 0, 2)
    try:
        assert full.acc_mode() == 1 and red.acc_mode() == 2
        assert red.device_bytes() < full.device_bytes()
    finally:
        full.free()
        red.free()


def test_config_values(L):
    """-1 is refused; 0 and nwin both give full tables; a value above nwin also does."""
    from gosnark_b200 import _lib
    assert L.b200_config(CFG_TABLE_WINDOWS, -1) == EINVAL
    n = 1 << 12
    c = adv.pick_window_bits(n)
    nwin = adv.n_windows(c)
    _, pool = adv.base_pool(1, "equal", c, seed=1)
    for t in (0, nwin, nwin + 5):
        bs = load(1, pool, n, 0, t)
        try:
            assert bs.table_windows() == nwin, t
        finally:
            bs.free()
    t = ctypes.c_int(0)
    assert L.b200_bases_table_windows(0, ctypes.byref(t)) == EINVAL


def _launches(L, fn):
    from gosnark_b200._lib import check
    buf = (ctypes.c_double * 8)()
    check(L.b200_profile_read(buf))
    fn()
    check(L.b200_profile_read(buf))
    return int(buf[6])


@pytest.mark.parametrize("g,logn", [(1, 14), (2, 11)])
def test_grouped_tail_adds_no_launch(L, g, logn):
    """With c >= 7 an MSM on a reduced set issues at most one launch more than on the full set, same kernel (XYZZ)."""
    n = 1 << logn
    c = adv.pick_window_bits(n)
    assert c >= 7
    ks, pool = adv.base_pool(g, "pm-pairs", c, seed=9)
    s = adv.full_width(n, np.random.default_rng(1))
    full = load(g, pool, n, 2, 0)
    counts = {}
    try:
        counts[0] = _launches(L, lambda: full.msm(limbs=s))
        for t in (1, 3):
            red = load(g, pool, n, 2, t)
            try:
                counts[t] = _launches(L, lambda: red.msm(limbs=s))
            finally:
                red.free()
    finally:
        full.free()
    assert all(counts[t] <= counts[0] + 1 for t in (1, 3)), counts


def _table_bytes(n, g):
    """window-table bytes of a full set of n points minus those of a t = 1 set"""
    c = adv.pick_window_bits(n)
    return (adv.n_windows(c) - 1) * n * (64 if g == 1 else 128)


# ---- proving keys -------------------------------------------------------------------------------------------------------
SIZES = [(1 << 12) + 2, 1 << 16]


def load_pk(syn, t, rank=0, world=1, ctx=0):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check, lib
    check(lib().b200_config(_lib.CFG_PK_CONTEXT, ctx))
    try:
        with _lib.table_windows(t):
            return syn.load_pk(rank, world)
    finally:
        check(lib().b200_config(_lib.CFG_PK_CONTEXT, 0))


def _dev(limbs):
    import torch
    return torch.from_numpy(np.ascontiguousarray(limbs).reshape(-1).view(np.int64)).cuda()


def _expected(syn, w_ints):
    a, b, c = syn.expected_dlogs(witness=w_ints, r=syn.r, s=syn.s)
    return G1.affine(G1.mul_scalar(G1.G, a)), G2.affine(G2.mul_scalar(G2.G, b)), G1.affine(G1.mul_scalar(G1.G, c))


def _affine(p):
    return G1.affine(p[0]), G2.affine(p[1]), G1.affine(p[2])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", SIZES, ids=["4098", "65536"])
def test_groth16_reduced_keys(L, deg_instances, n):
    """t = 1 and t = 3: b200_groth16_prove, _prove_witness, _prove_witness_device and _prove_device return the
    known-discrete-log proof, equal to the full-table key's, which verifies with its public signal and not with another."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    syn = deg.instance("groth16", n)
    w_ints = deg.chain_witness(n, R - 1)
    w = ints_to_limbs(w_ints)
    px = syn.px_of(w)
    exp = _expected(syn, w_ints)
    full = load_pk(syn, 0)
    try:
        pa, pb, pc = np.zeros(12, np.uint64), np.zeros(24, np.uint64), np.zeros(12, np.uint64)
        rr, ss = ptr(deg.limbs(syn.r)), ptr(deg.limbs(syn.s))
        check(L.b200_groth16_prove(full, ptr(w), syn.m, ptr(px), px.shape[0], rr, ss, ptr(pa), ptr(pb), ptr(pc)))
        assert _affine(deg.split(np.concatenate([pa, pc, pb]))) == exp
        for t in (1, 3):
            pk = load_pk(syn, t)
            try:
                deg.check_groth16_entry_points(L, syn, pk, w_ints, px, f"t={t}")
                d_out = torch.full((48,), -1, dtype=torch.int64, device="cuda")
                d_w, d_px = _dev(w), _dev(px)
                torch.cuda.synchronize()
                check(L.b200_groth16_prove_device(pk, d_w.data_ptr(), syn.m, d_px.data_ptr(), px.shape[0], rr, ss,
                                                  d_out.data_ptr(), None))
                torch.cuda.synchronize()
                assert _affine(deg.split(d_out.cpu().numpy().view(np.uint64))) == exp, t
            finally:
                check(L.b200_pk_free(pk))
    finally:
        check(L.b200_pk_free(full))


@pytest.mark.timeout(900)
def test_reduced_key_device_bytes(L, deg_instances):
    """At 2^20 constraints a t = 1 key holds at least the saved window-table bytes less than the full key.  (At small n
    the t = 1 key's G bucket arrays, a per-key constant, can outweigh the saving.)"""
    from gosnark_b200._lib import check, pk_device_bytes
    syn = deg.instance("groth16", 1 << 20)
    sets = [(syn.m + 3, 1), (syn.m + 3, 1), (syn.m + 3, 2), (syn.m - syn.npublic - 1 + syn.n_ptd + 1, 1)]
    predicted = sum(_table_bytes(k, g) for k, g in sets)
    full = load_pk(syn, 0)
    try:
        full_bytes = pk_device_bytes(full)
    finally:
        check(L.b200_pk_free(full))
    red = load_pk(syn, 1)
    try:
        red_bytes = pk_device_bytes(red)
    finally:
        check(L.b200_pk_free(red))
    assert full_bytes - red_bytes >= predicted, (full_bytes, red_bytes, predicted)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [2, 3])
def test_groth16_reduced_sharded_keys(L, deg_instances, world):
    """Ranks of a t = 1 key sharded 2 and 3 ways each prove from the device witness; the finalized records are the
    known-discrete-log proof."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    n = (1 << 12) + 2
    syn = deg.instance("groth16", n)
    w_ints = deg.chain_witness(n, R - 1)
    d_w = _dev(ints_to_limbs(w_ints))
    rr, ss = ptr(deg.limbs(syn.r)), ptr(deg.limbs(syn.s))
    pks = [load_pk(syn, 1, rank=rk, world=world) for rk in range(world)]
    try:
        parts = torch.zeros(128 * world, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        for rk, pk in enumerate(pks):
            check(L.b200_groth16_prove_witness_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, rr, ss,
                                                      parts[128 * rk:].data_ptr(), None))
        d_out = torch.zeros(48, dtype=torch.int64, device="cuda")
        check(L.b200_groth16_finalize_device(pks[0], parts.data_ptr(), world, rr, ss, d_out.data_ptr(), None))
        torch.cuda.synchronize()
        assert _affine(deg.split(d_out.cpu().numpy().view(np.uint64))) == _expected(syn, w_ints)
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
def test_two_contexts_in_flight_on_reduced_keys(L, deg_instances):
    """Keys with t = 1 (context 0) and t = 3 (context 1) prove at once on two streams; both proofs are exact."""
    import torch
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    n = 1 << 16
    syn = deg.instance("groth16", n)
    w_ints = deg.chain_witness(n, R - 1)
    d_w = _dev(ints_to_limbs(w_ints))
    rr, ss = ptr(deg.limbs(syn.r)), ptr(deg.limbs(syn.s))
    pks = [load_pk(syn, 1, ctx=0), load_pk(syn, 3, ctx=1)]
    try:
        outs = [torch.full((48,), -1, dtype=torch.int64, device="cuda") for _ in pks]
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        for _ in range(2):
            for pk, out, st in zip(pks, outs, streams):
                check(L.b200_groth16_prove_witness_device(pk, syn.r1cs.handle, d_w.data_ptr(), syn.m, rr, ss,
                                                          out.data_ptr(), st.cuda_stream))
        for st in streams:
            st.synchronize()
        exp = _expected(syn, w_ints)
        for out in outs:
            assert _affine(deg.split(out.cpu().numpy().view(np.uint64))) == exp
    finally:
        for pk in pks:
            check(L.b200_pk_free(pk))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", SIZES, ids=["4098", "65536"])
def test_pinocchio_reduced_keys(L, deg_instances, n):
    """b200_pinocchio_prove on t = 1 and t = 3 keys: all eight elements are the known discrete logs and the proof
    verifies under the real Vk."""
    from gosnark_b200._lib import check, ints_to_limbs, ptr
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    syn = deg.instance("pinocchio", n)
    order = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")
    w_ints = deg.chain_witness(n, R - 1)
    w = ints_to_limbs(w_ints)
    px = syn.px_of(w)
    exp = syn.expected_dlogs(w_ints)
    for t in (1, 3):
        pk = load_pk(syn, t)
        try:
            g1, pb = np.zeros(84, np.uint64), np.zeros(24, np.uint64)
            check(L.b200_pinocchio_prove(pk, ptr(w), syn.m, ptr(px), px.shape[0], ptr(g1), ptr(pb)))
            proof = dict(zip(order, _unflatten_g1(g1)))
            proof["PiB"] = _unflatten_g2(pb)[0]
            for k in order:
                assert G1.affine(proof[k]) == G1.affine(G1.mul_scalar(G1.G, exp[k])), (t, k)
            assert G2.affine(proof["PiB"]) == G2.affine(G2.mul_scalar(G2.G, exp["PiB"])), t
            assert syn.verify(proof, [w_ints[1]]), t
        finally:
            check(L.b200_pk_free(pk))


@pytest.fixture(scope="module")
def deg_instances():
    yield
    for syn in deg._made.values():
        syn.r1cs.free()
    deg._made.clear()
