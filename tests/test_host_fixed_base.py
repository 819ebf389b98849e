"""CPU: the fixed-base kernel of the sparse trusted setup (csrc/fixed_base.cuh) and its generator table, run through the
library's own orchestration (fixed_base_mul) over emulated kernels (tests/host/fixed_base_test.cpp, csrc/host_stub).
For G1 and G2, every output is the oracle's affine k*G: edge scalars, scalars whose signed digits are the extreme
values +2^(c-1) and -(2^(c-1) - 1), scalars whose top window receives a carry, and random full-width scalars."""
import ctypes
import random

import numpy as np
import pytest

import build as b200build
from oracle import ref_py as o

R_ = o.R


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_fixed_base())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _scalars(c):
    """Edge cases first, then digit extremes, top-window carries and random values; all < r."""
    half, nwin = 1 << (c - 1), (255 + c - 1) // c
    top = (nwin - 1) * c                                     # first bit of the top window
    ks = [0, 1, 2, R_ - 1, 1 << 253, half, half - 1, half + 1, (1 << c) - 1]
    # every window's digit +2^(c-1) (raw value half, no carry), and every digit -(half - 1) (raw half + 1)
    ks.append(sum(half << (c * w) for w in range(nwin - 1)) % R_)
    ks.append(sum((half + 1) << (c * w) for w in range(nwin - 1)) % R_)
    # a negative digit in the window below the top one carries into the top window
    for low in (half + 1, (1 << c) - 1):
        ks.append((low << (top - c)) | (1 << top))
        ks.append((low << (top - c)) + (R_ >> top << top) - (1 << top))   # just under r's top bits
    rng = random.Random(20261015)
    ks += [rng.randrange(R_) for _ in range(16)]
    for k in ks:
        assert 0 <= k < R_
    return ks


@pytest.mark.parametrize("group", [1, 2])
def test_fixed_base_equals_oracle(lib, group):
    c = lib.t_fixed_base_c()
    ks = _scalars(c)
    G = o.BN.G1 if group == 1 else o.BN.G2
    w = 8 if group == 1 else 16
    out = np.zeros(len(ks) * 3 * w, dtype=np.uint32)
    assert lib.t_fixed_base(group, _ptr(_u32(ks)), len(ks), _ptr(out)) == 0
    raw = out.tobytes()
    v = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(len(raw) // 32)]
    per = 3 if group == 1 else 6
    for i, k in enumerate(ks):
        p = v[per * i:per * (i + 1)]
        got = tuple(p) if group == 1 else ((p[0], p[1]), (p[2], p[3]), (p[4], p[5]))
        if k == 0:
            assert all(x == 0 for x in p), i
            continue
        e = G.affine(G.mul_scalar(G.G, k))
        assert got == ((e[0], e[1], 1) if group == 1 else (e[0], e[1], (1, 0))), (i, hex(k))


def test_scalars_reach_the_digit_extremes_and_the_top_carry(lib):
    """The inputs above really exercise what they claim, by the recode rule of for_each_digit."""
    c = lib.t_fixed_base_c()
    half, nwin = 1 << (c - 1), (255 + c - 1) // c
    seen_pos = seen_neg = seen_carry = False
    for k in _scalars(c):
        carry = 0
        for w in range(nwin):
            raw = ((k >> (w * c)) & ((1 << c) - 1)) + carry
            neg = raw > half
            d = raw - (1 << c) if neg else raw
            seen_pos |= d == half
            seen_neg |= d == -(half - 1)
            seen_carry |= w == nwin - 1 and carry == 1
            carry = int(neg)
        assert carry == 0                                   # no carry out of the top window for k < r
    assert seen_pos and seen_neg and seen_carry
