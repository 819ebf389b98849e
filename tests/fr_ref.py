"""Exact F_r references for the polynomial and QAP tests at scale: O(n) Python-int checks (Horner, the barycentric form of
the interpolant over {1..n}, Lagrange basis values by one batch inversion) and numpy limb helpers for inputs and exact
whole-output comparisons."""
import numpy as np

from oracle import ref_py as o

R = o.R
R_LIMBS = np.array([(R >> (64 * i)) & (2 ** 64 - 1) for i in range(4)], dtype=np.uint64)


def rand_limbs(n, seed):
    """n uniformly random residues < r as (n, 4) uint64 limbs (top limb drawn below r's, so every value is < r)."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2 ** 64, size=(n, 4), dtype=np.uint64, endpoint=False)
    a[:, 3] = rng.integers(0, int(R_LIMBS[3]), size=n, dtype=np.uint64)
    return a


def small_limbs(vals):
    """Non-negative integers < 2^64 as (n, 4) limbs."""
    a = np.zeros((len(vals), 4), dtype=np.uint64)
    a[:, 0] = np.asarray(vals, dtype=np.uint64)
    return a


def r_minus(vals):
    """r - v for integers 0 < v < 2^60 as limbs (r's low limb exceeds every v: no borrow)."""
    a = np.tile(R_LIMBS, (len(vals), 1))
    a[:, 0] -= np.asarray(vals, dtype=np.uint64)
    return a


def to_ints(a):
    raw = np.ascontiguousarray(a, dtype=np.uint64).tobytes()
    return [int.from_bytes(raw[i:i + 32], "little") for i in range(0, len(raw), 32)]


def from_ints(vals):
    buf = b"".join((int(v) % R).to_bytes(32, "little") for v in vals)
    return np.frombuffer(buf, dtype=np.uint64).reshape(len(vals), 4).copy()


def horner(c, x):
    acc = 0
    for v in reversed(c):
        acc = (acc * x + v) % R
    return acc


def batch_inv(xs):
    """[1/x for x in xs] (all non-zero mod r) with one modular inversion."""
    pre, acc = [], 1
    for x in xs:
        pre.append(acc)
        acc = acc * x % R
    inv = pow(acc, -1, R)
    out = [0] * len(xs)
    for i in range(len(xs) - 1, -1, -1):
        out[i] = inv * pre[i] % R
        inv = inv * xs[i] % R
    return out


_weights = {}


def weights(n):
    """Barycentric weights of the nodes 1..n: w_j = (-1)^(n-j) / ((j-1)! (n-j)!), j = 1..n (list index j - 1), and n!."""
    if n not in _weights:
        fact = [1] * (n + 1)
        for i in range(1, n + 1):
            fact[i] = fact[i - 1] * i % R
        invf = [1] * (n + 1)
        invf[n] = pow(fact[n], -1, R)
        for i in range(n, 0, -1):
            invf[i - 1] = invf[i] * i % R
        w = [invf[j - 1] * invf[n - j] % R for j in range(1, n + 1)]
        for j in range(n - 1, 0, -2):          # (-1)^(n-j) < 0: j = n-1, n-3, ...
            w[j - 1] = R - w[j - 1] if w[j - 1] else 0
        _weights.clear()                       # one n at a time: the lists are large
        _weights[n] = (w, fact[n])
    return _weights[n]


def zero_at(n, tau):
    """Z(tau) = prod_{i=1..n} (tau - i)."""
    acc = 1
    for i in range(1, n + 1):
        acc = acc * (tau - i) % R
    return acc


def lagrange_at(n, tau):
    """[l_j(tau) for j = 1..n]: the Lagrange basis of the nodes 1..n at tau (tau not a node) = Z(tau) w_j / (tau - j)."""
    w, _ = weights(n)
    z = zero_at(n, tau)
    inv = batch_inv([(tau - j) % R for j in range(1, n + 1)])
    return [z * wj % R * ij % R for wj, ij in zip(w, inv)]


def interp_at(vals, lag):
    """The interpolant of vals (at the nodes 1..n) evaluated where lag was taken: sum_j v_j l_j."""
    return sum(v * l for v, l in zip(vals, lag)) % R


def top_coeff(vals):
    """x^(n-1) coefficient of the interpolant of vals over 1..n: sum_j v_j w_j."""
    w, _ = weights(len(vals))
    return sum(v * x for v, x in zip(vals, w)) % R


def spmv(csr, w):
    """[sum_k val[k] w[col[k]] for each row] of one CSR matrix (rowptr, col, val limbs) and a witness of ints."""
    rowptr, col, val = csr
    vals = to_ints(val)
    out = []
    for j in range(len(rowptr) - 1):
        acc = 0
        for k in range(int(rowptr[j]), int(rowptr[j + 1])):
            acc += vals[k] * w[int(col[k])]
        out.append(acc % R)
    return out


def check_qap_px(csr, w, abc_px, tau, nodes):
    """(ax, bx, cx, px) limbs of b200_qap_px for witness w: ax, bx, cx are the interpolants over 1..n of A w, B w, C w (checked
    at tau against the barycentric sum), px(tau) = ax(tau) bx(tau) - cx(tau), and px vanishes at `nodes` when w satisfies
    the R1CS.  Returns px as ints."""
    n = len(csr[0][0]) - 1
    lag = lagrange_at(n, tau)
    ev = []
    for M, got in zip(csr, abc_px[:3]):
        c = to_ints(got)
        assert len(c) == n
        e = horner(c, tau)
        assert e == interp_at(spmv(M, w), lag), "interpolant of the matrix-witness product at tau"
        ev.append(e)
    px = to_ints(abc_px[3])
    assert len(px) == 2 * n - 1
    assert horner(px, tau) == (ev[0] * ev[1] - ev[2]) % R, "px(tau) != ax(tau) bx(tau) - cx(tau)"
    for j in nodes:
        assert horner(px, j) == 0, f"px({j}) != 0 for a satisfying witness"
    return px
