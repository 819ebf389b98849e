"""CPU: the kernels of batched proving on Groth16 key shards on the emulated threads (tests/host/shard_batch_test.cpp over
csrc/host_stub), with the launch shapes the library uses.

- k_groth16_finalize_batch over world x k partial records, laid out rank-major as an all-gather of k records per rank
  leaves them, equals k runs of the single proof's finalisation (the same kernel with k = 1, over each proof's world
  records) bit for bit, and each point is the sum of its records.  Records at infinity, records equal to each other (the
  doubling case of xyzz_add) and records that cancel are included.
- The C||PTD scalar vectors of a shard, w[l1 + c_lo ..) ++ h[p_lo, p_hi) ++ 0.. ++ [-r s] (the tail only on the rank that
  holds it), restated here, against k_quotient_store with a source offset.
- k_pinocchio_gather_finalize_batch over world x k Pinocchio records, rank-major, equals k runs of the single proof's
  gather-finalisation (the same kernel with k = 1) bit for bit, and each point is the sum of its records, with the same
  cases.
- The ptxas report of the library build shows no spills in the kernels this feature adds or changed."""
import ctypes
import os
import random
import re

import numpy as np
import pytest

import build as b200build
from oracle import ref_py as o

R_, Q_ = o.R, o.Q
G1, G2 = o.BN.G1, o.BN.G2


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_shard_batch())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ints(a, cnt):
    raw = a.tobytes()
    return [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(cnt)]


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _records(rng, world, k):
    """dlogs[(g, p, slot)] for slots A, B1, C (G1) and B2 (G2); None is infinity.  Proof 0 has a record at infinity on
    every slot of rank 0, proof 1 two equal records (rank 0 and 1), proof 2 two that cancel, the rest random."""
    d = {}
    for g in range(world):
        for p in range(k):
            for slot in ("A", "B1", "C", "B2"):
                d[(g, p, slot)] = rng.randrange(1, R_)
    for slot in ("A", "B1", "C", "B2"):
        if k > 0:
            d[(0, 0, slot)] = None
            if world > 2:
                d[(world - 1, 0, slot)] = None
        if k > 1 and world > 1:
            d[(1, 1, slot)] = d[(0, 1, slot)]
        if k > 2 and world > 1:
            d[(world - 1, 2, slot)] = (R_ - d[(0, 2, slot)]) % R_
    return d


def _pt(G, x):
    return None if x is None else G.affine(G.mul_scalar(G.G, x))


def _sum(G, dlogs):
    """The affine sum of the records, from their discrete logs (None: infinity); None when it is infinity."""
    t = sum(x for x in dlogs if x is not None) % R_
    return None if t == 0 else G.affine(G.mul_scalar(G.G, t))


@pytest.mark.parametrize("k", [1, 5])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_finalize_batch_equals_single_finalize(lib, world, k):
    rng = random.Random(1000 * world + k)
    d = _records(rng, world, k)
    nrec = world * k
    g1 = {}
    g2 = {}
    for g in range(world):
        for p in range(k):
            for slot in ("A", "B1", "C"):
                g1[(g, p, slot)] = _pt(G1, d[(g, p, slot)])
            g2[(g, p)] = _pt(G2, d[(g, p, "B2")])
    xy1, xy2 = [], []
    for e in range(nrec):
        g, p = divmod(e, k)
        for slot in ("A", "B1", "C"):
            pt = g1[(g, p, slot)]
            xy1 += [0, 0] if pt is None else list(pt[:2])
        pt = g2[(g, p)]
        xy2 += [0, 0, 0, 0] if pt is None else [c for xy in pt[:2] for c in xy]
    scale = [rng.randrange(1, Q_) for _ in range(3 * nrec)] + [c for _ in range(nrec) for c in (rng.randrange(1, Q_), rng.randrange(Q_))]
    out_b = np.zeros(8 * 12 * k, dtype=np.uint32)
    out_s = np.zeros(8 * 12 * k, dtype=np.uint32)
    assert lib.t_groth16_finalize_batch(_ptr(_u32(xy1)), _ptr(_u32(xy2)), _ptr(_u32(scale)), world, k, _ptr(out_b), _ptr(out_s)) == 0
    assert out_b.tobytes() == out_s.tobytes()          # bit for bit: the batch is k single finalisations
    words = _ints(out_b, 12 * k)
    for p in range(k):
        w = words[12 * p:12 * p + 12]
        for j, slot in ((0, "A"), (1, "C")):
            want = _sum(G1, [d[(g, p, slot)] for g in range(world)])
            X, Y, Z = w[3 * j:3 * j + 3]
            if want is None:
                assert Z == 0, (slot, p)
            else:
                assert Z != 0 and tuple(G1.affine((X, Y, Z))[:2]) == tuple(want[:2]), (slot, p)
        want = _sum(G2, [d[(g, p, "B2")] for g in range(world)])
        X, Y, Z = ([w[6 + 2 * i], w[7 + 2 * i]] for i in range(3))
        if want is None:
            assert Z == [0, 0], p
        else:
            assert tuple(tuple(c) for c in G2.affine((X, Y, Z))[:2]) == tuple(tuple(c) for c in want[:2]), p


def shard_ch_vectors(ws, hs, neg_rs, l1, c_lo, n_c, p_lo, n_p, tail):
    """A shard's C||PTD scalar vectors, restated: w_p[l1 + c_lo, l1 + c_lo + n_c) ++ h_p[p_lo, p_lo + n_p) (zero beyond
    len(h_p)) ++ [-r_p s_p] when the rank holds the tail."""
    out = []
    for w, h, t in zip(ws, hs, neg_rs):
        out += w[l1 + c_lo:l1 + c_lo + n_c]
        out += [h[i] if i < len(h) else 0 for i in range(p_lo, p_lo + n_p)]
        out += [t] if tail else []
    return out


@pytest.mark.parametrize("with_coef", [True, False], ids=["h-direct", "in-place"])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("cut", ["whole", "c-and-head", "middle", "tail-past-h", "tail-only-zeros"])
def test_quotient_store_with_offset(lib, cut, k, with_coef):
    rng = random.Random(f"{cut}/{k}/{with_coef}")
    m, l1 = 40, 2
    ncf = m - l1
    nh, n_ptd = 33, m - 1                         # len(h) < len(PTD): the zero fill
    c_lo, c_hi, p_lo, p_hi = {"whole": (0, ncf, 0, n_ptd), "c-and-head": (10, ncf, 0, 12), "middle": (ncf, ncf, 5, 20),
                              "tail-past-h": (ncf, ncf, 20, n_ptd), "tail-only-zeros": (ncf, ncf, 35, n_ptd)}[cut]
    tail = p_hi == n_ptd
    n_c, n_p = c_hi - c_lo, p_hi - p_lo
    stride = n_c + n_p + (1 if tail else 0)
    ws = [[rng.randrange(R_) for _ in range(m)] for _ in range(k)]
    hs = [[rng.randrange(R_) for _ in range(nh)] for _ in range(k)]
    neg_rs = [rng.randrange(R_) for _ in range(k)]
    want = shard_ch_vectors(ws, hs, neg_rs, l1, c_lo, n_c, p_lo, n_p, tail)
    cstride = nh + 5
    coef = [v for h in hs for v in h + [rng.randrange(R_) for _ in range(cstride - nh)]]
    vec = []
    for p in range(k):                            # the C slice copied already; the quotient part garbage or in place
        row = ws[p][l1 + c_lo:l1 + c_hi] + [rng.randrange(R_) for _ in range(stride - n_c)]
        if not with_coef:
            have = max(0, min(nh - p_lo, n_p))
            row[n_c:n_c + have] = hs[p][p_lo:p_lo + have]
        vec += row
    buf = _u32(vec)
    tl = _u32(neg_rs) if tail else None
    assert lib.t_quotient_store_shard(_ptr(_u32(coef)) if with_coef else None, cstride, nh, p_lo, n_p,
                                      _ptr(tl) if tail else None, k, stride, n_c, _ptr(buf)) == 0
    assert _ints(buf, k * stride) == want


PIN_SLOTS = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


@pytest.mark.parametrize("k", [1, 5])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_pinocchio_gather_finalize_batch_equals_single(lib, world, k):
    """Each slot of a proof is owned by one rank in the library, but the kernel sums every rank's record; here every
    record is set, so the sums cover infinity, doubling and cancelling records as well."""
    rng = random.Random(7000 + 100 * world + k)
    nrec = world * k
    d = {}
    for g in range(world):
        for p in range(k):
            for s in PIN_SLOTS + ("PiB",):
                d[(g, p, s)] = rng.randrange(1, R_)
    for s in PIN_SLOTS + ("PiB",):
        d[(0, 0, s)] = None
        if k > 1 and world > 1:
            d[(1, 1, s)] = d[(0, 1, s)]
        if k > 2 and world > 1:
            d[(world - 1, 2, s)] = (R_ - d[(0, 2, s)]) % R_
    xy1, xy2 = [], []
    for e in range(nrec):
        g, p = divmod(e, k)
        for s in PIN_SLOTS:
            pt = _pt(G1, d[(g, p, s)])
            xy1 += [0, 0] if pt is None else list(pt[:2])
        pt = _pt(G2, d[(g, p, "PiB")])
        xy2 += [0, 0, 0, 0] if pt is None else [c for xy in pt[:2] for c in xy]
    scale = [rng.randrange(1, Q_) for _ in range(7 * nrec)] + [c for _ in range(nrec) for c in (rng.randrange(1, Q_), rng.randrange(Q_))]
    out_b = np.zeros(8 * 27 * k, dtype=np.uint32)
    out_s = np.zeros(8 * 27 * k, dtype=np.uint32)
    assert lib.t_pinocchio_gather_finalize_batch(_ptr(_u32(xy1)), _ptr(_u32(xy2)), _ptr(_u32(scale)), world, k, _ptr(out_b),
                                                 _ptr(out_s)) == 0
    assert out_b.tobytes() == out_s.tobytes()
    words = _ints(out_b, 27 * k)
    for p in range(k):
        w = words[27 * p:27 * p + 27]
        for i, s in enumerate(PIN_SLOTS):
            want = _sum(G1, [d[(g, p, s)] for g in range(world)])
            X, Y, Z = w[3 * i:3 * i + 3]
            if want is None:
                assert Z == 0, (s, p)
            else:
                assert Z != 0 and tuple(G1.affine((X, Y, Z))[:2]) == tuple(want[:2]), (s, p)
        want = _sum(G2, [d[(g, p, "PiB")] for g in range(world)])
        X, Y, Z = ([w[21 + 2 * i], w[22 + 2 * i]] for i in range(3))
        if want is None:
            assert Z == [0, 0], p
        else:
            assert tuple(tuple(c) for c in G2.affine((X, Y, Z))[:2]) == tuple(tuple(c) for c in want[:2]), p


NEW_KERNELS = ["k_groth16_finalize_batch", "k_groth16_fold_products_batch", "k_quotient_store", "k_pinocchio_records_batch",
               "k_pinocchio_gather_finalize_batch"]


def test_new_kernels_do_not_spill():
    """ptxas (-Xptxas -v, sm_90a) of the library build: no spill stores or loads in the kernels this feature adds or
    changed."""
    b200build.build_cuda()
    log = os.path.join(b200build.LIBDIR, "nvcc_build.log")
    if not os.path.exists(log):
        pytest.skip("the library was not built here (no ptxas report)")
    text = open(log).read()
    blocks = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'.*?\n(?:.*\n)*?.*?(\d+) bytes spill stores, (\d+) bytes spill loads",
                        text)
    seen = set()
    for mangled, st, ld in blocks:
        for name in NEW_KERNELS:
            if re.search(r"\d%s" % name + r"[A-Z_]", mangled) or mangled.endswith(name):
                seen.add(name)
                assert (int(st), int(ld)) == (0, 0), (name, st, ld)
    assert seen == set(NEW_KERNELS), set(NEW_KERNELS) - seen
