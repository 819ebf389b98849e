// CPU test vehicle for the setup straight into a resident key (g++, csrc/host_stub): the library's own minting path —
// FixedBaseTable::build, fixed_base_row_enqueue into a base set's row 0, then window_table_enqueue from that row — over
// emulated kernels, one thread at a time; and the per-rank set plan of both key kinds (shard_partition.h).  Test
// infrastructure only: never linked into libb200snark.
#include "host_stub/cuda_runtime.h"

#include <vector>

template <class K> void stub_launch_threads(unsigned nblocks, unsigned nthreads, K k);
#define B200_LAUNCH(kernel, grid, block, stream, ...) stub_launch_threads((unsigned)(grid), (unsigned)(block), [&] { kernel(__VA_ARGS__); })
#define B200_LAUNCH_CTA(kernel, grid, block, stream, ...) stub_abort("CTA kernel")
#include "fixed_base.cuh"
#include "shard_partition.h"

using namespace b200;

// none of the kernels run here synchronises inside a CTA
void stub_syncthreads() { stub_abort("__syncthreads"); }
uint32_t stub_shfl(uint32_t, int, int, int) { stub_abort("warp shuffle"); }
void stub_syncwarp() {}
unsigned stub_ballot(int) { stub_abort("__ballot_sync"); }

template <class K>
void stub_launch_threads(unsigned nblocks, unsigned nthreads, K kernel) {
  blockDim.x = nthreads;
  gridDim.x = nblocks;
  for (unsigned b = 0; b < nblocks; b++)
    for (unsigned t = 0; t < nthreads; t++) {
      blockIdx.x = b;
      threadIdx.x = t;
      kernel();
    }
}

namespace {
template <class F>
int mint_table(const uint32_t* scalars_std, uint32_t n, int c, uint32_t rows, uint32_t* table_out) {
  std::vector<Fr> s(n);
  std::memcpy(s.data(), scalars_std, (size_t)n * sizeof(Fr));
  std::vector<Affine<F>> table((size_t)rows * n);
  std::vector<XYZZ<F>> state(n);
  int err = 0;
  FixedBaseTable<F> gen;
  if (gen.build(&err, nullptr)) return 1;
  fixed_base_row_enqueue<F>(gen, s.data(), n, table.data(), state.data(), nullptr);
  window_table_enqueue<F>(nullptr, n, rows, c, table.data(), state.data(), &err, nullptr);
  std::memcpy(table_out, table.data(), table.size() * sizeof(Affine<F>));
  return err ? 100 + err : 0;
}
// The two-step path to the same table: the host setup's standard-form points (fixed_base_std), then the load's
// k_load_bases and window rows.
template <class F>
int load_table(const uint32_t* scalars_std, uint32_t n, int c, uint32_t rows, uint32_t* table_out) {
  std::vector<Fr> s(n);
  std::memcpy(s.data(), scalars_std, (size_t)n * sizeof(Fr));
  std::vector<F> pts((size_t)3 * n);
  std::vector<Affine<F>> table((size_t)rows * n);
  std::vector<XYZZ<F>> state(n);
  int err = 0;
  FixedBaseTable<F> gen;
  if (gen.build(&err, nullptr) || fixed_base_std<F>(gen, s.data(), n, pts.data(), nullptr)) return 1;
  window_table_enqueue<F>(pts.data(), n, rows, c, table.data(), state.data(), &err, nullptr);
  std::memcpy(table_out, table.data(), table.size() * sizeof(Affine<F>));
  return err ? 100 + err : 0;
}
}  // namespace

extern "C" {
// table_out = rows x n Montgomery affine points (x | y), row w holding 2^(c*w) * k_i * G; infinity all zero.  group 1 = G1,
// 2 = G2.  rows: the key's stored window rows (all ceil(255/c) of them, or t of a reduced table).
int t_mint_table(int group, const uint32_t* scalars_std, uint32_t n, int c, uint32_t rows, uint32_t* table_out) {
  return group == 1 ? mint_table<Fq>(scalars_std, n, c, rows, table_out) : mint_table<Fq2>(scalars_std, n, c, rows, table_out);
}
// the same table through the host setup's points and the load's k_load_bases
int t_load_table(int group, const uint32_t* scalars_std, uint32_t n, int c, uint32_t rows, uint32_t* table_out) {
  return group == 1 ? load_table<Fq>(scalars_std, n, c, rows, table_out) : load_table<Fq2>(scalars_std, n, c, rows, table_out);
}
// Groth16 set plan of rank `rank`: out = lo[4] | hi[4] | tail[4] | len[4]
int t_groth16_plan(uint64_t m, uint64_t npublic, uint64_t n_ptd, const double wgt[4], int rank, int world, uint64_t* out) {
  G16Plan p = groth16_set_plan((size_t)m, (size_t)npublic, (size_t)n_ptd, wgt, rank, world);
  for (int k = 0; k < 4; k++) {
    out[k] = p.cuts[(size_t)rank].lo[k];
    out[4 + k] = p.cuts[(size_t)rank].hi[k];
    out[8 + k] = p.tail[k];
    out[12 + k] = p.len[k];
  }
  return 0;
}
// Pinocchio dealing: owner[k] of the eight sets
int t_pinocchio_owners(uint64_t m, uint64_t l1, uint64_t n_g1t, int world, int* owner) {
  pinocchio_owners((size_t)m, (size_t)l1, (size_t)n_g1t, world, owner);
  return 0;
}
}
