"""CPU: the index-range partition of a sharded Groth16 key (csrc/shard_partition.h, compiled with g++ behind a C entry
point) against its Python mirror (gosnark_b200/shard.py), and the properties the multi-GPU decomposition rests on:
every set is tiled exactly once in rank order and no rank's weighted load exceeds the equal share by more than a term
per set."""
import ctypes
import os
import random
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def cpart():
    import build
    lib = ctypes.CDLL(build.build_shard_partition())
    lib.shard_partition_c.restype = ctypes.c_int

    def run(lens, wgt, world):
        l = np.array(lens, dtype=np.uint64)
        w = np.array(wgt, dtype=np.float64)
        out = np.zeros(8 * world, dtype=np.uint64)
        lib.shard_partition_c(l.ctypes.data_as(ctypes.c_void_p), w.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(world),
                              out.ctypes.data_as(ctypes.c_void_p))
        o = out.reshape(world, 4, 2)
        return [([int(o[g, k, 0]) for k in range(4)], [int(o[g, k, 1]) for k in range(4)]) for g in range(world)]
    return run


def cases():
    rng = random.Random(11)
    out = [((1 << 20) + 2, 1, (1 << 20) + 1, w) for w in (1, 2, 3, 4, 8)]
    out += [((1 << 16) + 2, 1, (1 << 16) + 1, w) for w in (2, 8)]
    out += [(66, 1, 65, w) for w in (2, 3, 8, 64, 200)]          # more ranks than terms: empty ranks
    for _ in range(80):
        m = rng.randrange(3, 5000)
        out.append((m, rng.randrange(0, min(m - 1, 4)), rng.randrange(1, 5000), rng.randrange(1, 17)))
    return out


@pytest.mark.parametrize("w_ab,w_g2", [(1.0, 2.8), (0.85, 2.75), (1.3, 3.3)])
def test_cpp_partition_equals_python_mirror_and_tiles(cpart, w_ab, w_g2):
    from gosnark_b200 import shard
    for m, npublic, n_ptd, world in cases():
        lens = (m, m, m, m - npublic - 1 + n_ptd)
        wgt = (w_ab, w_ab, w_g2, 1.0)
        got = cpart(lens, wgt, world)
        exp = shard.partition(lens, wgt, world)
        assert got == [(list(lo), list(hi)) for lo, hi in exp], (m, world)
        for k in range(4):                      # exact tiling in rank order
            pos = 0
            for lo, hi in got:
                assert lo[k] <= hi[k] <= lens[k]
                if lo[k] < hi[k]:
                    assert lo[k] == pos
                    pos = hi[k]
            assert pos == lens[k], (m, world, k)
        load = [sum(wgt[k] * (hi[k] - lo[k]) for k in range(4)) for lo, hi in got]
        ideal = sum(w * l for w, l in zip(wgt, lens)) / world
        assert max(load) <= ideal + 4 * max(wgt) + 1e-9


def test_shard_ranges_defaults_are_the_recorded_partition():
    """The default weights reproduce the recorded cuts of the 8-rank split of a 2^20-constraint key (witness ranges)."""
    from gosnark_b200 import shard
    m = (1 << 20) + 2
    s1 = shard.shard_ranges(m, 1, (1 << 20) + 1, 1, 8)["sets"]
    assert (s1[0]["lo"], s1[0]["hi"], s1[1]["lo"], s1[1]["hi"]) == (891290, 1048578, 0, 734003)
    s7 = shard.shard_ranges(m, 1, (1 << 20) + 1, 7, 8)["sets"]
    assert (s7[3]["lo"], s7[3]["hi"], s7[3]["tail"]) == (1205862, 2097153, True)
