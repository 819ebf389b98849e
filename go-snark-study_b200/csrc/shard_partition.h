// Index-range partition of the four MSMs of a Groth16 proving key (A, B1, B2, C||PTD) over `world` ranks
// (SURVEY §8e; groth16/groth16.go:241-270 are the four sums).  Plain C++ — no CUDA — so that the CPU suite can
// compile it with g++ and hold it against its Python mirror (go-snark-study_b200/shard.py, tests/test_shard_partition.py).
//
// The sets lie end to end on a line weighted by cost per term (wgt[k], in G1 terms of the C||PTD set) and the line is
// cut into `world` equal pieces: rank g holds whole sets where it can and an index range where it must; rank g's `lo`
// is rank g-1's `hi`, so every set is tiled exactly once.
// (Measured and dropped: a fixed cost per piece with greedy filling to the smallest
// common capacity.  The ranks that hold two pieces are the FAST ones — their two MSMs fill each other's gaps.)
#pragma once
#include <cstddef>

namespace b200 {

struct ShardCut {
  size_t lo[4], hi[4];
};

// cuts[g] for g in [0, world)
inline void shard_partition(const size_t len[4], const double wgt[4], int world, ShardCut* cuts) {
  double off[5] = {0, 0, 0, 0, 0};
  for (int k = 0; k < 4; k++) off[k + 1] = off[k] + wgt[k] * (double)len[k];
  auto cut = [&](int g, int k) -> size_t {   // first index of set k at or after the g-th cut of the line
    if (g >= world) return len[k];
    double pos = off[4] * (double)g / (double)world;
    double x = (pos - off[k]) / wgt[k];
    if (x <= 0) return 0;
    if (x >= (double)len[k]) return len[k];
    return (size_t)x;
  };
  for (int g = 0; g < world; g++)
    for (int k = 0; k < 4; k++) {
      cuts[g].lo[k] = cut(g, k);
      cuts[g].hi[k] = cut(g + 1, k);
    }
}

}  // namespace b200
