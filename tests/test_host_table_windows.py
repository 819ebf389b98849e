"""CPU: MSMs over reduced window tables (B200_CFG_TABLE_WINDOWS) through the library's MSM engine (msm_host.cuh) on the
CPU emulation (tests/host/table_windows_test.cpp, csrc/host_stub): the library's table build with t rows, the grouped signed-digit recode
and counting sort, both accumulation kernels, the grouped tails and the Horner chain over all window groups.  Every result
is the oracle's sum_i s_i * P_i, for G1 and G2, t in {1, 2, 5, nwin - 1, nwin} and c below and above the c = 7 switch
between the segment tail and the rows / columns / planes tail."""
import ctypes
import random

import numpy as np
import pytest

import build as b200build
from oracle import ref_py as o

R_ = o.R


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_table_windows())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _flat(pts):
    flat = []
    for p in pts:
        for cc in p:
            flat.extend(cc if isinstance(cc, tuple) else (cc,))
    return flat


def _point(group, out):
    raw = out.tobytes()
    v = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(len(raw) // 32)]
    return (v[0], v[1], v[2]) if group == 1 else ((v[0], v[1]), (v[2], v[3]), (v[4], v[5]))


def _expect(group, k):
    G = o.BN.G1 if group == 1 else o.BN.G2
    if k % R_ == 0:
        return (0, 0, 0) if group == 1 else ((0, 0), (0, 0), (0, 0))
    e = G.affine(G.mul_scalar(G.G, k % R_))
    return (e[0], e[1], 1) if group == 1 else (e[0], e[1], (1, 0))


def _digits(k, c):
    """for_each_digit restated: [(window, signed digit)] and the carry into each window."""
    half, nwin = 1 << (c - 1), (255 + c - 1) // c
    carry, out, carries = 0, [], []
    for w in range(nwin):
        raw = ((k >> (w * c)) & ((1 << c) - 1)) + carry
        carries.append(carry)
        neg = raw > half
        out.append(raw - (1 << c) if neg else raw)
        carry = int(neg)
    assert carry == 0
    return out, carries


def _boundary_scalars(c, t):
    """Scalars whose last window of a group has a negative digit, so the carry enters the first window of the next group."""
    nwin = (255 + c - 1) // c
    ks = []
    for w0 in (t - 1, 2 * t - 1, nwin - 2):
        if t >= nwin or w0 + 1 >= nwin or (w0 + 1) % t:
            continue
        for low in ((1 << c) - 1, (1 << (c - 1)) + 1):
            ks.append((low << (w0 * c)) + (1 << ((w0 + 1) * c)))
    return ks


def _scalars(rng, c, t, n):
    sc = [0, 1, R_ - 1] + _boundary_scalars(c, t)
    sc += [rng.randrange(R_) for _ in range(n - len(sc))]
    return sc[:n]


CASES = [(1, 4, 0), (1, 5, 8), (1, 7, 0), (1, 8, 16), (2, 5, 0), (2, 7, 0)]


@pytest.mark.parametrize("group,c,S", CASES)
@pytest.mark.parametrize("which_t", ["1", "2", "5", "nwin-1", "nwin"])
def test_reduced_table_msm_equals_oracle(lib, group, c, S, which_t):
    nwin = (255 + c - 1) // c
    t = {"1": 1, "2": 2, "5": 5, "nwin-1": nwin - 1, "nwin": nwin}[which_t]
    G = o.BN.G1 if group == 1 else o.BN.G2
    n = 24 if group == 1 else 12
    rng = random.Random(100 * group + 10 * c + t)
    ks = [rng.randrange(1, R_) for _ in range(n)]
    ks[3] = ks[4]                                           # a repeated point
    pts = [G.mul_scalar(G.G, k) for k in ks]                # Jacobian, Z != 1
    sc = _scalars(rng, c, t, n)
    w = 8 if group == 1 else 16
    out = np.zeros(3 * w, dtype=np.uint32)
    assert lib.t_msm_grouped(group, _ptr(_u32(_flat(pts))), _ptr(_u32(sc)), n, c, t, S, _ptr(out)) == 0
    assert _point(group, out) == _expect(group, sum(k * s for k, s in zip(ks, sc)))


@pytest.mark.parametrize("c", [4, 5, 7, 8, 9])
@pytest.mark.parametrize("t", [1, 2, 5])
def test_boundary_scalars_carry_across_groups(c, t):
    """The boundary scalars really carry out of the last window of one group into the first window of the next."""
    nwin = (255 + c - 1) // c
    ks = _boundary_scalars(c, t)
    assert ks
    for k in ks:
        assert 0 <= k < R_
        digits, carries = _digits(k, c)
        crossing = [w for w in range(1, nwin) if w % t == 0 and carries[w] == 1 and digits[w - 1] < 0]
        assert crossing, (c, t, hex(k))


@pytest.mark.parametrize("group", [1, 2])
@pytest.mark.parametrize("nplanes,groups,gshift", [(6, 1, 0), (8, 1, 0), (6, 5, 7), (8, 3, 18), (16, 15, 17), (6, 37, 7)])
def test_horner_over_groups(lib, group, nplanes, groups, gshift):
    """k_tail_horner alone: sum_g 2^(g*gshift) (sum_j 2^j P_g[j] + P_g[nplanes]) for planes of known discrete logs."""
    G = o.BN.G1 if group == 1 else o.BN.G2
    rng = random.Random(nplanes * 1000 + groups * 10 + group)
    logs = [rng.randrange(1, R_) for _ in range(groups * (nplanes + 1))]
    logs[0] = logs[-1] = 0                                  # planes at infinity
    flat = []
    for k in logs:
        if k == 0:
            flat += [0, 0] if group == 1 else [0, 0, 0, 0]
        else:
            a = G.affine(G.mul_scalar(G.G, k))
            flat += [a[0], a[1]] if group == 1 else [*a[0], *a[1]]
    exp = 0
    for g in range(groups):
        P = logs[g * (nplanes + 1):(g + 1) * (nplanes + 1)]
        exp += (sum(P[j] << j for j in range(nplanes)) + P[nplanes]) << (g * gshift)
    w = 8 if group == 1 else 16
    out = np.zeros(3 * w, dtype=np.uint32)
    assert lib.t_tail_horner(group, _ptr(_u32(flat)), nplanes, groups, gshift, _ptr(out)) == 0
    assert _point(group, out) == _expect(group, exp)
