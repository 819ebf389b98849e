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
#include <algorithm>
#include <cstddef>
#include <vector>

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

// Whether the rank whose cut of set k is [lo, hi) also holds the set's blinding points (its tail): the rank holding the
// set's last element, or, if no rank holds elements of it (len == 0), the last rank.
inline bool shard_holds_tail(size_t lo, size_t hi, size_t len, int rank, int world) {
  return hi == len && (lo < hi || (rank == world - 1 && len == 0));
}

// The set plan of a Groth16 key for rank `rank` of `world`: the lengths of its four sets (A, B1, B2: m; C||PTD:
// m - npublic - 1 + n_ptd), every rank's cut of them (wgt: the cost per term of each set), and which tails this rank holds.
struct G16Plan {
  size_t len[4];
  std::vector<ShardCut> cuts;
  bool tail[4];
};
inline G16Plan groth16_set_plan(size_t m, size_t npublic, size_t n_ptd, const double wgt[4], int rank, int world) {
  G16Plan p;
  const size_t len[4] = {m, m, m, m - npublic - 1 + n_ptd};
  p.cuts.resize((size_t)world);
  shard_partition(len, wgt, world, p.cuts.data());
  for (int k = 0; k < 4; k++) {
    p.len[k] = len[k];
    p.tail[k] = shard_holds_tail(p.cuts[(size_t)rank].lo[k], p.cuts[(size_t)rank].hi[k], len[k], rank, world);
  }
  return p;
}

// The eight base sets of a sharded Pinocchio key (0 A, 1 Ap, 2 B (G2), 3 Bp, 4 C, 5 Cp, 6 Kp, 7 G1T) are independent
// objects, so whole sets are dealt to the ranks: greedy longest-first onto the least loaded rank by term count (a G2 term
// ~2.8 G1 terms), and no set is split.  owner[k] is the same on every rank; more than 8 ranks leave the rest idle.
inline void pinocchio_owners(size_t m, size_t l1, size_t n_g1t, int world, int owner[8]) {
  double cost[8] = {(double)(m - l1), (double)(m - l1), 2.8 * (double)m, (double)m, (double)m, (double)m, (double)m, (double)n_g1t};
  int order[8] = {0, 1, 2, 3, 4, 5, 6, 7};
  std::stable_sort(order, order + 8, [&](int x, int y) { return cost[x] > cost[y]; });
  std::vector<double> load((size_t)world, 0.0);
  for (int q = 0; q < 8; q++) {
    int k = order[q], best = 0;
    for (int g = 1; g < world; g++)
      if (load[g] < load[best]) best = g;
    owner[k] = best;
    load[best] += cost[k];
  }
}

}  // namespace b200
