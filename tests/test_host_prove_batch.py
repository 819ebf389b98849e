"""CPU: the batched QAP front end of b200_groth16_prove_witness_batch (csrc/qap_sparse.cuh) on the emulated kernels
(tests/host/prove_batch_test.cpp over csrc/host_stub).

- qap_h_batch gives the k quotients that k runs of the single-witness qap_h_from_values give, bit for bit, satisfied
  value sets or not, and for small n the oracle's DivisorPolynomial(ax*bx - cx, Z).
- k_spmm_ab (one thread per row and tile of witnesses) equals k_spmv_csr per witness on irregular CSR.
- The scalar-vector layouts of a batch: W_p = w_p ++ [1, r_p, s_p] and C||PTD_p = w_p[l+1..m) ++ h_p ++ 0.. ++ [-r_p s_p],
  restated here, against k_quotient_store.
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
    return ctypes.CDLL(b200build.build_host_prove_batch())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ints(a, cnt):
    raw = a.tobytes()
    return [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(cnt)]


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _value_sets(n, k, seed):
    """k value sets (a, b, c) on {1..n}: satisfied ones next to one row off, every row off and c = 0."""
    rng = random.Random(seed)
    hows = ["sat", "one", "every", "c=0", "sat", "last", "one"]
    out = []
    for p in range(k):
        a = [rng.randrange(R_) for _ in range(n)]
        b = [rng.randrange(R_) for _ in range(n)]
        c = [x * y % R_ for x, y in zip(a, b)]
        how = hows[p % len(hows)]
        if how == "one":
            c[n // 2] = (c[n // 2] + 1) % R_
        elif how == "last":
            c[-1] = (c[-1] + 7) % R_
        elif how == "every":
            c = [rng.randrange(R_) for _ in range(n)]
        elif how == "c=0":
            c = [0] * n
        out.append((a, b, c))
    return out


@pytest.mark.parametrize("k", [1, 2, 3, 7])
@pytest.mark.parametrize("n", [2, 3, 5, 17, 64, 257, 1500])
def test_batched_quotients_equal_single_ones(lib, n, k):
    sets = _value_sets(n, k, 1000 * n + k)
    flat = [v for a, b, c in sets for v in a + b + c]
    hb = np.zeros(8 * k * (n - 1) + 8, dtype=np.uint32)
    hs = np.zeros_like(hb)
    assert lib.t_qap_h_batch(_ptr(_u32(flat)), n, k, _ptr(hb), _ptr(hs)) == 0
    assert np.array_equal(hb, hs)
    if n <= 40:
        z = [1]
        for i in range(1, n + 1):
            z = o.PF.mul(z, [(-i) % R_, 1])
        got = _ints(hb, k * (n - 1))
        for p, (a, b, c) in enumerate(sets):
            ax, bx, cx = (o.PF.lagrange_interpolation(v) for v in (a, b, c))
            exp = o.PF.divisor_polynomial(o.PF.sub(o.PF.mul(ax, bx), cx), z)
            assert got[p * (n - 1):(p + 1) * (n - 1)] == exp, p


def _irregular_csr(n, m, rng):
    """CSR with empty rows, a 512-term row, explicit 0 and r-1 coefficients, and repeated (row, column) entries."""
    rows = []
    for j in range(n):
        kind = j % 5
        if kind == 0:
            rows.append([])
        elif kind == 1:
            rows.append([(rng.randrange(m), rng.choice([0, R_ - 1, 1]))])
        elif kind == 2:
            c = rng.randrange(m)
            rows.append([(c, rng.randrange(R_)), (c, rng.randrange(R_)), (c, R_ - 1)])
        else:
            rows.append([(rng.randrange(m), rng.randrange(R_)) for _ in range(rng.randrange(1, 6))])
    rows[n // 2] = [(rng.randrange(m), rng.randrange(R_)) for _ in range(512)]
    rowptr, col, val = [0], [], []
    for r in rows:
        for c, v in r:
            col.append(c)
            val.append(v)
        rowptr.append(len(col))
    return np.array(rowptr, np.uint32), np.array(col or [0], np.uint32), _u32(val or [0]), rows


@pytest.mark.parametrize("k", [1, 3, 4, 5, 6, 9])
def test_sparse_product_over_k_witnesses(lib, k):
    n, m = 37, 23
    rng = random.Random(k)
    A, B = _irregular_csr(n, m, rng), _irregular_csr(n, m, rng)
    w = [rng.randrange(R_) for _ in range(k * m)]
    out = np.zeros(8 * 3 * k * n, dtype=np.uint32)
    ref = np.zeros_like(out)
    err = ctypes.c_int(0)
    assert lib.t_spmm_ab(n, m, _ptr(A[0]), _ptr(A[1]), _ptr(A[2]), _ptr(B[0]), _ptr(B[1]), _ptr(B[2]), _ptr(_u32(w)), k,
                         _ptr(out), _ptr(ref), ctypes.byref(err)) == 0
    assert err.value == 0
    assert np.array_equal(out, ref)
    got = _ints(out, 3 * k * n)
    for p in range(k):       # and the sums themselves, from the rows
        wp = w[p * m:(p + 1) * m]
        av = [sum(v * wp[c] for c, v in A[3][j]) % R_ for j in range(n)]
        bv = [sum(v * wp[c] for c, v in B[3][j]) % R_ for j in range(n)]
        assert got[3 * p * n:(3 * p + 1) * n] == av
        assert got[(3 * p + 1) * n:(3 * p + 2) * n] == bv
        assert got[(3 * p + 2) * n:(3 * p + 3) * n] == [x * y % R_ for x, y in zip(av, bv)]


def test_witness_entry_out_of_range_reads_as_zero(lib):
    n, m, k = 5, 4, 3
    rowptr = np.array([0, 1, 2, 3, 4, 4], np.uint32)
    col = np.array([0, 1, 2, 3], np.uint32)
    val = _u32([1, 1, 1, 1])
    w = [5, 6, 7, 8, 9, 10, R_, 12, 13, 14, 15, 16]
    out = np.zeros(8 * 3 * k * n, dtype=np.uint32)
    ref = np.zeros_like(out)
    err = ctypes.c_int(0)
    assert lib.t_spmm_ab(n, m, _ptr(rowptr), _ptr(col), _ptr(val), _ptr(rowptr), _ptr(col), _ptr(val), _ptr(_u32(w)), k,
                         _ptr(out), _ptr(ref), ctypes.byref(err)) == 0
    assert err.value & 2
    got = _ints(out, 3 * k * n)
    assert got[3 * n:3 * n + n] == [9, 10, 0, 12, 0]


def batch_vectors(ws, rs_pairs, l1, hs, n_ptd):
    """The scalar vectors of a batch, restated: W_p (stride m + 3) and C||PTD_p (stride (m - l1) + n_ptd + 1)."""
    W, CH = [], []
    for w, (r, s), h in zip(ws, rs_pairs, hs):
        W += list(w) + [1, r, s]
        CH += list(w[l1:]) + list(h) + [0] * (n_ptd - len(h)) + [(-r * s) % R_]
    return W, CH


@pytest.mark.parametrize("with_coef", [True, False])
def test_quotient_store_builds_the_c_ptd_vectors(lib, with_coef):
    rng = random.Random(3)
    k, m, l1, nh, n_ptd = 4, 9, 3, 5, 8
    ws = [[rng.randrange(R_) for _ in range(m)] for _ in range(k)]
    hs = [[rng.randrange(R_) for _ in range(nh)] for _ in range(k)]
    rs = [(rng.randrange(R_), rng.randrange(R_)) for _ in range(k)]
    W, CH = batch_vectors(ws, rs, l1, hs, n_ptd)
    assert len(W) == k * (m + 3) and W[(m + 3) + m:(m + 3) + m + 3] == [1, *rs[1]]
    nc, stride = m - l1, m - l1 + n_ptd + 1
    # what the library holds before the store: the C parts copied, garbage (or, with_coef False, h) after them
    vec = []
    for p in range(k):
        rest = [rng.randrange(R_) for _ in range(n_ptd + 1)]
        if not with_coef:
            rest[:nh] = hs[p]
        vec += ws[p][l1:] + rest
    cstride = 8
    coef = [v for h in hs for v in h + [0] * (cstride - nh)]
    small = [v for r, s in rs for v in (1, r, s, (-r * s) % R_)]    # the batch's {1, r_p, s_p, -r_p s_p}
    tail = _u32(small[3:] + [0, 0, 0])                              # read from its fourth entry, stride 4
    buf = _u32(vec)
    assert lib.t_quotient_store(_ptr(_u32(coef)) if with_coef else None, cstride, nh, n_ptd, _ptr(tail), 4, k, _ptr(buf),
                                stride, nc) == 0
    assert _ints(buf, k * stride) == CH


NEW_KERNELS = ["k_witness_load_batch", "k_spmm_ab", "k_take_blocks", "k_quotient_store", "k_groth16_products_batch",
               "k_groth16_combine_batch", "k_newton_scale", "k_h_values"]


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
