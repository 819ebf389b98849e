"""GPU: the sparse QAP front end (qap_sparse.cuh / qap_sparse_host.cuh behind b200_interpolate, b200_zero_poly, b200_qap_px,
b200_qap_eval_at) at the sizes the prove path and the trusted setup use, against exact Python-int references.

The kernel path changes with the size: the subproduct tree over N = pow2 >= n (schoolbook levels below 16 points,
transforms above; n = 2^k + 1 doubles the tree), batched transforms that tile only when the total is a multiple of 1024,
the one-block Z kernel up to 2048 roots and the tree above.  The references are O(n): the barycentric form of the
interpolant over {1..n} with one batch inversion, Horner, and the closed forms of Z's extreme coefficients.  The last test
is one sequence that shrinks, regrows and revisits sizes, so that the caches kept across calls (transform plans and
workspaces, the domains by N, the e^(-x) series, a divisor's inverse) are read at sizes other than the ones that built
them."""
import random

import numpy as np
import pytest

from fr_ref import R, check_qap_px, from_ints, horner, interp_at, lagrange_at, rand_limbs, to_ints, top_coeff, weights, zero_at

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


def interpolate(L, v):
    from gosnark_b200._lib import check, ptr
    out = np.zeros_like(v)
    check(L.b200_interpolate(ptr(v), v.shape[0], ptr(out)))
    return out


def edge_values(n, seed):
    """Random values with zeros, small integers and r - 1 among them, at both ends as well."""
    v = to_ints(rand_limbs(n, seed))
    rng = random.Random(seed)
    for j, x in zip([0, n - 1] + rng.sample(range(n), min(n, 30)), [0, R - 1] + [0, 1, 5, R - 1] * 8):
        v[j] = x
    return v


def check_interpolant(coeffs, v, seed):
    """coeffs is the interpolant of v over {1..n}: at random tau against the barycentric sum, exactly at sampled nodes
    (1 and n always), and its top coefficient against sum_j v_j w_j."""
    n = len(v)
    c = to_ints(coeffs)
    assert len(c) == n
    rng = random.Random(seed)
    for t in [rng.randrange(n + 1, R) for _ in range(1 if n > (1 << 18) + 1 else 2)]:
        assert horner(c, t) == interp_at(v, lagrange_at(n, t)), ("tau", n, t)
    for j in sorted({1, n} | set(rng.sample(range(1, n + 1), min(n, 2 if n > (1 << 18) + 1 else 6)))):
        assert horner(c, j) == v[j - 1], ("node", n, j)
    assert c[n - 1] == top_coeff(v), ("top coefficient", n)


INTERP_N = [255, 256, 257, 511, 512, 513, (1 << 18) - 1, 1 << 18, (1 << 18) + 1, (1 << 20) + 1, 1 << 22]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", INTERP_N)
def test_interpolate(L, n):
    v = edge_values(n, n)
    check_interpolant(interpolate(L, from_ints(v)), v, n)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [2048, 2049, (1 << 20) - 1, (1 << 20) + 1, 1 << 22])
def test_zero_poly(L, n):
    """Z = prod_{i=1..n}(x - i) (the one-block kernel at 2048, the tree above): Z(tau) at a random tau, Z(i) = 0 at sampled
    roots (n included), and the closed forms: monic, x^(n-1) coefficient -n(n+1)/2, constant (-1)^n n!."""
    from gosnark_b200._lib import check, ptr
    z = np.zeros((n + 1, 4), dtype=np.uint64)
    check(L.b200_zero_poly(n, ptr(z)))
    zc = to_ints(z)
    rng = random.Random(n)
    t = rng.randrange(n + 1, R)
    assert horner(zc, t) == zero_at(n, t)
    for i in sorted({1, n, rng.randrange(2, n)}):
        assert horner(zc, i) == 0, i
    assert zc[n] == 1
    assert zc[n - 1] == (-(n * (n + 1) // 2)) % R
    _, fact_n = weights(n)
    assert zc[0] == (fact_n if n % 2 == 0 else R - fact_n)


def circuit(n, seed=None):
    from gosnark_b200.synthetic import SyntheticCircuit
    return SyntheticCircuit(n) if seed is None else SyntheticCircuit(n, seed=seed)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [(1 << 17) + 1, 1 << 20, (1 << 20) + 1])
def test_qap_px(L, n):
    """b200_qap_px on the synthetic chain: ax, bx, cx are the interpolants of A w, B w, C w (computed in Python from the
    CSR), px = ax bx - cx vanishes at the nodes for the satisfying witness; after x_k += 1 the row that defines x_k reads
    x_{k-1} x_{k-2} - (x_k + 1) = -1, so px(k) = r - 1 exactly."""
    from gosnark_b200._lib import ints_to_limbs
    from gosnark_b200.r1csqap import SparseR1CS
    circ = circuit(n)
    sp = SparseR1CS(n, circ.m, circ.csr)
    try:
        rng = random.Random(n)
        out = sp.combine_limbs(ints_to_limbs(circ.witness))
        check_qap_px(circ.csr, circ.witness, out, rng.randrange(n + 1, R), sorted({1, n, rng.randrange(2, n)}))
        k = n // 2
        w2 = list(circ.witness)
        w2[2 + k] = (w2[2 + k] + 1) % R
        px2 = to_ints(sp.combine_limbs(ints_to_limbs(w2), want_abc=False)[3])
        assert horner(px2, k) == R - 1
    finally:
        sp.free()


def eval_at_reference(csr, n, m, tau):
    """[sum_j M[j][i] l_j(tau) for each signal i] for the three matrices, and Z(tau) over the n nodes."""
    lag = lagrange_at(n, tau)
    outs = []
    for rowptr, col, val in csr:
        vals = to_ints(val)
        acc = [0] * m
        for j in range(n):
            for k in range(int(rowptr[j]), int(rowptr[j + 1])):
                acc[int(col[k])] += vals[k] * lag[j]
        outs.append([x % R for x in acc])
    return outs, zero_at(n, tau)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("tau", ["n+1", "r-1", "random"])
@pytest.mark.parametrize("n", [(1 << 17) + 1, 1 << 20])
def test_qap_eval_at(L, n, tau):
    """b200_qap_eval_at: Eval(alphas[i], tau) etc. for every signal through A^T l(tau), and Z(tau)."""
    from gosnark_b200.r1csqap import SparseR1CS
    circ = circuit(n)
    t = {"n+1": n + 1, "r-1": R - 1, "random": random.Random(n).randrange(n + 1, R)}[tau]
    sp = SparseR1CS(n, circ.m, circ.csr)
    try:
        at, bt, ct, zt = sp.EvalAt(t)
    finally:
        sp.free()
    exp, ez = eval_at_reference(circ.csr, n, circ.m, t)
    assert [to_ints(at), to_ints(bt), to_ints(ct)] == exp
    assert zt == ez


# One sequence, in this order: products, divisions and interpolations that shrink, regrow and revisit sizes after
# everything above (and, in a full run, the 2^27 product of test_gpu_poly_scale.py) has grown the caches.
ORDER = [("mul", 1 << 22), ("mul", 1 << 9), ("mul", (1 << 19) + 1),
         ("div", 1 << 20), ("div", 1 << 10), ("div", (1 << 20) + 1),
         ("interpolate", (1 << 20) + 1), ("interpolate", 1 << 21), ("interpolate", 300)]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("op,size", ORDER, ids=[f"{i}-{op}-{s}" for i, (op, s) in enumerate(ORDER)])
def test_order_shrink_regrow_revisit(L, op, size):
    from gosnark_b200._lib import check, ptr
    rng = random.Random(size)
    if op == "mul":
        na = size // 2 + 1
        a, b = rand_limbs(na, size), rand_limbs(size - na + 1, size + 1)
        out = np.zeros((size, 4), dtype=np.uint64)
        check(L.b200_poly_mul(ptr(a), a.shape[0], ptr(b), b.shape[0], ptr(out)))
        t = rng.randrange(R)
        assert horner(to_ints(out), t) == horner(to_ints(a), t) * horner(to_ints(b), t) % R
    elif op == "div":
        nb = 33
        a, b = rand_limbs(size + nb - 1, size), rand_limbs(nb, size + 1)
        b[nb - 1, 0] |= np.uint64(1)
        q, rem = np.zeros((size, 4), dtype=np.uint64), np.zeros((nb - 1, 4), dtype=np.uint64)
        check(L.b200_poly_div(ptr(a), a.shape[0], ptr(b), nb, ptr(q), ptr(rem)))
        t = rng.randrange(R)
        assert horner(to_ints(a), t) == (horner(to_ints(q), t) * horner(to_ints(b), t) + horner(to_ints(rem), t)) % R
    else:
        v = edge_values(size, size + 7)
        check_interpolant(interpolate(L, from_ints(v)), v, size + 7)
