"""CPU: the quotient by len(Z) = n of witness-fed proving on circuits with m = n + 1 signals (csrc/qap_sparse.cuh:
k_short_z_lambda, k_short_z_dot, k_quotient_store_shifted after the batched front end), on the emulated kernels
(tests/host/short_z_test.cpp over csrc/host_stub).

- The scalar vectors the batch writes hold DivisorPolynomial(ax*bx - cx, Z_n) with Z_n = prod_{i=1..n-1}(x - i), exactly,
  for satisfied and unsatisfied witnesses, k in {1, 3, 8}, and from shard offsets p_lo > 0 (a slice starting past len(h)
  included), with the tail after them.
- The launches the library counts for the branch do not depend on k.
- The ptxas report of the library build shows no spills in the new kernels."""
import ctypes
import os
import random
import re

import numpy as np
import pytest

import build as b200build
from oracle import ref_py as o

R_ = o.R


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_short_z())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ints(a, cnt):
    raw = a.tobytes()
    return [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(cnt)]


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---- Python-int restatements, O(n^2): the oracle's own routines are O(n^3) and serve the small sizes -----------------
def _interpolate(v):
    """LagrangeInterpolation over x = 1..n: Newton forward differences, then the Newton basis expanded."""
    n = len(v)
    d, cur = [], list(v)
    for k in range(n):
        d.append(cur[0] * pow(_fact(k), -1, R_) % R_)
        cur = [(cur[i + 1] - cur[i]) % R_ for i in range(len(cur) - 1)]
    out, basis = [0] * n, [1]                          # basis = prod_{i=1..k}(x - i)
    for k in range(n):
        for i, c in enumerate(basis):
            out[i] = (out[i] + d[k] * c) % R_
        basis = _mul(basis, [(-(k + 1)) % R_, 1])
    return out


def _fact(k):
    f = 1
    for i in range(2, k + 1):
        f = f * i % R_
    return f


def _mul(a, b):
    out = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        if x:
            for j, y in enumerate(b):
                out[i + j] = (out[i + j] + x * y) % R_
    return out


def _divisor_polynomial(px, z):
    """Long division by monic z with the remainder dropped (r1csqap.go:70-84, 213-216)."""
    rem, nz = list(px), len(z)
    q = [0] * (len(px) - nz + 1)
    for pos in range(len(q) - 1, -1, -1):
        c = rem[pos + nz - 1]
        q[pos] = c
        for i in range(nz):
            rem[pos + i] = (rem[pos + i] - c * z[i]) % R_
    return q


def _z(nroots):
    z = [1]
    for i in range(1, nroots + 1):
        z = _mul(z, [(-i) % R_, 1])
    return z


def _rows_csr(rows):
    rowptr, col, val = [0], [], []
    for r in rows:
        for c, v in r:
            col.append(c)
            val.append(v)
        rowptr.append(len(col))
    return np.array(rowptr, np.uint32), np.array(col or [0], np.uint32), _u32(val or [0])


def _matvec(rows, w):
    return [sum(v * w[c] for c, v in r) % R_ for r in rows]


def _circuit(n, m, rng):
    """A random sparse R1CS with empty rows, repeated columns and r - 1 coefficients."""
    def row(j):
        kind = j % 4
        if kind == 0 and j:
            return []
        if kind == 1:
            c = rng.randrange(m)
            return [(c, rng.randrange(R_)), (c, R_ - 1)]
        return [(rng.randrange(m), rng.randrange(R_)) for _ in range(rng.randrange(1, 4))]
    return [[row(j) for j in range(n)] for _ in range(3)]


def _reference_h(mats, w, n):
    av, bv, cv = (_matvec(M, w) for M in mats)
    ax, bx, cx = (_interpolate(v) for v in (av, bv, cv))
    px = [(x - (cx[i] if i < n else 0)) % R_ for i, x in enumerate(_mul(ax, bx))]
    return _divisor_polynomial(px, _z(n - 1))


def _satisfy(mats, w, n):
    """Make w satisfy row j of the R1CS by giving C's row j one more term on "one" (signal 0): C w then equals A w . B w."""
    A, B, C = mats
    av, bv, cv = (_matvec(M, w) for M in mats)
    for j in range(n):
        C[j] = C[j] + [(0, (av[j] * bv[j] - cv[j]) % R_)]


def _run(lib, mats, n, m, ws, n_ptd, off, stride):
    k = len(ws)
    csr = [_rows_csr(M) for M in mats]
    tail = [R_ - 1 - p for p in range(k)]
    vec = _u32([7] * (k * stride))
    lam = np.zeros(8 * n, np.uint32)
    launches = ctypes.c_ulonglong(0)
    err = ctypes.c_int(0)
    args = [a for c in csr for a in map(_ptr, c)]
    assert lib.t_short_z_batch(n, m, *args, _ptr(_u32([v for w in ws for v in w])), k, n_ptd, off, _ptr(_u32(tail)), _ptr(vec),
                               stride, _ptr(lam), ctypes.byref(launches), ctypes.byref(err)) == 0
    assert err.value == 0
    return _ints(vec, k * stride), tail, _ints(lam, n), launches.value


@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("n", [2, 3, 5, 64, 300])
def test_quotient_by_short_z_equals_divisor_polynomial(lib, n, k):
    rng = random.Random(1000 * n + k)
    m = n + 1
    mats = _circuit(n, m, rng)
    ws = [[1] + [rng.randrange(R_) for _ in range(m - 1)] for _ in range(k)]
    satisfied = k > 1 or n % 2 == 1         # witness 0 satisfies the R1CS (k = 1: for odd n), the others almost surely not
    if satisfied:
        _satisfy(mats, ws[0], n)
    got, tail, lam, _ = _run(lib, mats, n, m, ws, n, 0, n + 1)
    for j in range(n):                      # the weights of the top divided difference over {1..n}
        assert lam[j] == (-1) ** (n - 1 - j) * pow(_fact(j) * _fact(n - 1 - j), -1, R_) % R_
    for p, w in enumerate(ws):
        exp = _reference_h(mats, w, n)
        assert len(exp) == n
        assert got[p * (n + 1):(p + 1) * (n + 1)] == exp + [tail[p]], p
    if n <= 5:                              # the Python restatements against the oracle's own routines
        for w in ws:
            av, bv, cv = (_matvec(M, w) for M in mats)
            ax, bx, cx = (o.PF.lagrange_interpolation(v) for v in (av, bv, cv))
            assert ax == _interpolate(av)
            ref = o.PF.divisor_polynomial(o.PF.sub(o.PF.mul(ax, bx), cx), _z(n - 1))
            assert ref == _reference_h(mats, w, n)
    if satisfied:                           # a satisfied witness: kappa = 0, h Z_n = px exactly
        sat = _reference_h(mats, ws[0], n)
        av, bv, cv = (_matvec(M, ws[0]) for M in mats)
        assert av and [x * y % R_ for x, y in zip(av, bv)] == cv
        ax, bx, cx = (_interpolate(v) for v in (av, bv, cv))
        px = [(x - (cx[i] if i < n else 0)) % R_ for i, x in enumerate(_mul(ax, bx))]
        assert _mul(sat, _z(n - 1)) == px


@pytest.mark.parametrize("n, n_ptd, off", [(5, 3, 0), (5, 3, 2), (5, 3, 4), (5, 2, 5), (5, 4, 7), (64, 20, 30), (64, 30, 50)])
def test_shard_slices_from_an_offset(lib, n, n_ptd, off):
    """A rank whose PowersTauDelta slice starts at p_lo = off: h[off .. off + n_ptd) (zeros at and past len(h) = n), and
    only global index 0 takes kappa."""
    rng = random.Random(n * 100 + off)
    m, k = n + 1, 3
    mats = _circuit(n, m, rng)
    ws = [[1] + [rng.randrange(R_) for _ in range(m - 1)] for _ in range(k)]
    got, tail, _, _ = _run(lib, mats, n, m, ws, n_ptd, off, n_ptd + 2)
    for p, w in enumerate(ws):
        h = _reference_h(mats, w, n) + [0] * (off + n_ptd)
        vec = got[p * (n_ptd + 2):(p + 1) * (n_ptd + 2)]
        assert vec[:n_ptd] == h[off:off + n_ptd], p
        assert vec[n_ptd] == tail[p]
        assert vec[n_ptd + 1] == 7          # the slot past the tail is not written


def test_launches_do_not_depend_on_k(lib):
    # n = 600: every transform of the front end (3k x 2N, N = 1024) is a whole number of 1024-element tiles for any k, so
    # its launches are the same for every k too (below that the passes of ntt_batched depend on the total size)
    n, m = 600, 601
    rng = random.Random(9)
    mats = _circuit(n, m, rng)
    counts = set()
    for k in (1, 3, 8):
        ws = [[1] + [rng.randrange(R_) for _ in range(m - 1)] for _ in range(k)]
        counts.add(_run(lib, mats, n, m, ws, n, 0, n + 1)[3])
    assert len(counts) == 1 and counts.pop() > 3


NEW_KERNELS = ["k_short_z_lambda", "k_short_z_dot", "k_quotient_store_shifted"]


def test_new_kernels_do_not_spill():
    """ptxas (-Xptxas -v, sm_90a) of the library build: no spill stores or loads in the kernels this branch adds."""
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
