"""CPU: the kernels of b200_pinocchio_prove_witness_batch on the emulated threads (tests/host/pinocchio_batch_test.cpp over
csrc/host_stub), with the launch shapes the library uses.

- The G1T scalar vectors of a batch, h_p ++ 0.. at stride len(G1T), restated here, against k_quotient_store with no tail
  element: from the batched front end's Montgomery blocks, and from quotients already in place (the px-and-division
  branch), with len(G1T) > len(h) and == len(h).
- k_pinocchio_finalize_batch: records with known affine values and Z != 1, infinity records included, to k x 108 words.
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
SLOTS = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_pinocchio_batch())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ints(a, cnt):
    raw = a.tobytes()
    return [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(cnt)]


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def g1t_vectors(hs, n_g1t):
    """The G1T scalar vectors of a batch, restated: h_p, then zeros up to len(G1T)."""
    return [v for h in hs for v in list(h) + [0] * (n_g1t - len(h))]


@pytest.mark.parametrize("with_coef", [True, False], ids=["h-direct", "in-place"])
@pytest.mark.parametrize("k", [1, 2, 3, 7])
@pytest.mark.parametrize("n", [2, 3, 5, 17, 64, 257])
def test_quotient_store_builds_the_g1t_vectors(lib, n, k, with_coef):
    rng = random.Random(100 * n + k)
    nh = n - 1                                           # len(h) of an n-constraint circuit with len(Z) = n + 1
    for n_g1t in (nh, nh + 1, nh + 6):                   # == len(h), one more (CircuitPinocchio), zero fill
        hs = [[rng.randrange(R_) for _ in range(nh)] for _ in range(k)]
        cstride = nh + 3                                 # the front end's blocks are wider than a quotient
        coef = [v for h in hs for v in h + [rng.randrange(R_) for _ in range(cstride - nh)]]
        vec = []
        for p in range(k):                               # before the store: garbage, or the quotient in place
            row = [rng.randrange(R_) for _ in range(n_g1t)]
            if not with_coef:
                row[:nh] = hs[p]
            vec += row
        buf = _u32(vec)
        assert lib.t_quotient_store_g1t(_ptr(_u32(coef)) if with_coef else None, cstride, nh, n_g1t, k, _ptr(buf)) == 0
        assert _ints(buf, k * n_g1t) == g1t_vectors(hs, n_g1t), n_g1t


def _f2(v):
    return [v[0], v[1]]


@pytest.mark.parametrize("k", [1, 2, 3, 9, 64, 65])
def test_finalize_batch_writes_k_proofs(lib, k):
    """Record (slot s, proof p) = dlog * G in XYZZ form with ZZ = u^2, ZZZ = u^3: proof p's word block holds the seven G1
    points in slot order and then PiB, each affine-equal to its point and with Z = u^3; an infinity record gives twelve
    (G2: twenty-four) zero words.  k = 65 runs two G1 blocks' worth of G2 threads past the first G2 block."""
    rng = random.Random(k)
    inf1 = {(rng.randrange(7), rng.randrange(k)) for _ in range(3)} | {(0, 0)}
    inf2 = {rng.randrange(k)} | ({k - 1} if k > 1 else set())
    a1 = {(s, p): ((0, 0) if (s, p) in inf1 else tuple(G1.affine(G1.mul_scalar(G1.G, rng.randrange(1, R_)))[:2]))
          for s in range(7) for p in range(k)}
    a2 = {p: (((0, 0), (0, 0)) if p in inf2 else tuple(tuple(c) for c in G2.affine(G2.mul_scalar(G2.G, rng.randrange(1, R_)))[:2]))
          for p in range(k)}
    u1 = {e: rng.randrange(1, Q_) for e in a1}
    u2 = {p: (rng.randrange(1, Q_), rng.randrange(Q_)) for p in a2}
    g1_xy = _u32([c for s in range(7) for p in range(k) for c in a1[(s, p)]])
    g2_xy = _u32([c for p in range(k) for xy in a2[p] for c in xy])
    scale = _u32([u1[(s, p)] for s in range(7) for p in range(k)] + [c for p in range(k) for c in u2[p]])
    out = np.zeros(8 * 27 * k, dtype=np.uint32)
    assert lib.t_pinocchio_finalize_batch(_ptr(g1_xy), _ptr(g2_xy), _ptr(scale), k, _ptr(out)) == 0
    words = _ints(out, 27 * k)
    f2 = o.BN.Fq2
    for p in range(k):
        proof = words[27 * p:27 * p + 27]
        for s in range(7):
            X, Y, Z = proof[3 * s:3 * s + 3]
            if (s, p) in inf1:
                assert (X, Y, Z) == (0, 0, 0), (SLOTS[s], p)
                continue
            assert Z == pow(u1[(s, p)], 3, Q_), (SLOTS[s], p)
            assert tuple(G1.affine((X, Y, Z))[:2]) == a1[(s, p)], (SLOTS[s], p)
        X, Y, Z = (_f2(proof[21 + 2 * i:23 + 2 * i]) for i in range(3))
        if p in inf2:
            assert (X, Y, Z) == ([0, 0], [0, 0], [0, 0]), p
            continue
        u = list(u2[p])
        assert f2.equal(Z, f2.mul(f2.square(u), u)), p
        assert tuple(tuple(c) for c in G2.affine((X, Y, Z))[:2]) == a2[p], p


NEW_KERNELS = ["k_quotient_store", "k_pinocchio_finalize_batch"]


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
