"""CPU: the setup straight into a resident proving key (csrc/fixed_base.cuh, csrc/shard_partition.h), through the library's
own code over emulated kernels (tests/host/setup_key_test.cpp, csrc/host_stub).

- Minting into a base set's row 0 and building the window rows from it: for G1 and G2, every table row j equals the
  oracle's 2^(c*j) * k * G, for full tables and for t = 1 and 3 stored rows, with the edge scalars of
  test_host_fixed_base.py and k = 0 (infinity, the all-zero words k_load_bases writes).
- The minted table is the two-step path's word for word: the host setup's standard-form points loaded by k_load_bases
  and the same window rows give the same Montgomery words.
- The per-rank set plan: the Groth16 ranges and tails equal gosnark_b200/shard.py, and the Pinocchio dealing equals a
  Python restatement, for world 1, 2, 3 and 8."""
import ctypes
import random

import numpy as np
import pytest

import build as b200build
from oracle import ref_py as o

R_, Q_ = o.R, o.Q
RINV = pow(1 << 256, -1, Q_)                 # Montgomery form: x_mont = x * 2^256 mod q


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_setup_key())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _scalars(c):
    """The edge cases of test_host_fixed_base.py (0, 1, r - 1, digit extremes, a top-window carry) and random values."""
    half, nwin = 1 << (c - 1), (255 + c - 1) // c
    top = (nwin - 1) * c
    ks = [0, 1, 2, R_ - 1, 1 << 253, half, half - 1, half + 1, (1 << c) - 1, 0]
    ks.append(sum(half << (c * w) for w in range(nwin - 1)) % R_)
    ks.append(sum((half + 1) << (c * w) for w in range(nwin - 1)) % R_)
    ks.append(((half + 1) << (top - c)) | (1 << top))
    rng = random.Random(20261018)
    ks += [rng.randrange(R_) for _ in range(5)]
    assert all(0 <= k < R_ for k in ks)
    return ks


def _raw_table(lib, fn, group, ks, c, rows):
    fe = 8 if group == 1 else 16                                 # u32 words per coordinate
    out = np.zeros(rows * len(ks) * 2 * fe, dtype=np.uint32)
    assert fn(group, _ptr(_u32(ks)), len(ks), c, rows, _ptr(out)) == 0
    return out


def _table(lib, group, ks, c, rows):
    raw = _raw_table(lib, lib.t_mint_table, group, ks, c, rows).tobytes()
    v = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(len(raw) // 32)]
    per = 2 if group == 1 else 4
    return [v[per * i:per * (i + 1)] for i in range(rows * len(ks))]


@pytest.mark.parametrize("group", [1, 2])
@pytest.mark.parametrize("c,t", [(10, 0), (8, 1), (9, 3)])
def test_minted_rows_equal_the_oracle(lib, group, c, t):
    nwin = (255 + c - 1) // c
    rows = t if 0 < t < nwin else nwin
    ks = _scalars(c)
    G = o.BN.G1 if group == 1 else o.BN.G2
    tab = _table(lib, group, ks, c, rows)
    for j in range(rows):
        for i, k in enumerate(ks):
            words = tab[j * len(ks) + i]
            if k == 0:
                assert all(x == 0 for x in words), (j, i)         # Affine::inf()
                continue
            assert all(x < Q_ for x in words), (j, i)             # canonical Montgomery words
            std = [x * RINV % Q_ for x in words]
            got = tuple(std) if group == 1 else ((std[0], std[1]), (std[2], std[3]))
            e = G.affine(G.mul_scalar(G.G, (k << (c * j)) % R_))
            assert got == (e[0], e[1]), (group, c, t, j, i, hex(k))


@pytest.mark.parametrize("group", [1, 2])
@pytest.mark.parametrize("c,t", [(10, 0), (9, 3)])
def test_minted_table_is_the_loaded_table_word_for_word(lib, group, c, t):
    nwin = (255 + c - 1) // c
    rows = t if 0 < t < nwin else nwin
    ks = _scalars(c)
    minted = _raw_table(lib, lib.t_mint_table, group, ks, c, rows)
    loaded = _raw_table(lib, lib.t_load_table, group, ks, c, rows)
    assert np.array_equal(minted, loaded)


def _pinocchio_owners(m, l1, n_g1t, world):
    """Greedy longest-first dealing of the eight sets (csrc/shard_partition.h: pinocchio_owners)."""
    cost = [m - l1, m - l1, 2.8 * m, m, m, m, m, n_g1t]
    order = sorted(range(8), key=lambda k: -cost[k])            # stable, as std::stable_sort
    load, owner = [0.0] * world, [0] * 8
    for k in order:
        best = min(range(world), key=lambda g: (load[g], g))
        owner[k] = best
        load[best] += cost[k]
    return owner


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_set_plans_equal_the_python_mirrors(lib, world):
    from gosnark_b200 import shard
    rng = random.Random(world)
    shapes = [((1 << 12) + 2, 1), ((1 << 16) + 2, 1), ((1 << 16) + 1, 1), (66, 1), (12, 3)]
    shapes += [(rng.randrange(3, 5000), rng.randrange(0, 3)) for _ in range(10)]
    for m, npub in shapes:
        n_ptd = m - 1
        wgt = np.array(shard.weights(world), dtype=np.float64)
        for rank in range(world):
            out = np.zeros(16, dtype=np.uint64)
            lib.t_groth16_plan(ctypes.c_uint64(m), ctypes.c_uint64(npub), ctypes.c_uint64(n_ptd), _ptr(wgt), rank, world, _ptr(out))
            exp = shard.shard_ranges(m, npub, n_ptd, rank, world)
            for k in range(4):
                s = exp["sets"][k]
                assert (int(out[k]), int(out[4 + k]), bool(out[8 + k])) == (s["lo"], s["hi"], s["tail"]), (m, rank, k)
            assert [int(x) for x in out[12:]] == [m, m, m, exp["n_c_full"] + n_ptd]
        owner = (ctypes.c_int * 8)()
        lib.t_pinocchio_owners(ctypes.c_uint64(m), ctypes.c_uint64(npub + 1), ctypes.c_uint64(m - 1), world, owner)
        assert list(owner) == _pinocchio_owners(m, npub + 1, m - 1, world), (m, world)
