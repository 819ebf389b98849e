// CPU test vehicle for the fixed-base kernel of fixed_base.cuh (g++, csrc/host_stub): the library's own orchestration
// (fixed_base_mul: generator multiples by k_mul_batch_ref, the MSM window table, k_fixed_base, k_batch_to_affine,
// k_affine_store_std) over emulated kernels, one thread at a time.  Test infrastructure only: never linked into
// libb200snark.
#include "host_stub/cuda_runtime.h"

#include <vector>

template <class K> void stub_launch_threads(unsigned nblocks, unsigned nthreads, K k);
#define B200_LAUNCH(kernel, grid, block, stream, ...) stub_launch_threads((unsigned)(grid), (unsigned)(block), [&] { kernel(__VA_ARGS__); })
#define B200_LAUNCH_CTA(kernel, grid, block, stream, ...) stub_abort("CTA kernel")
#include "fixed_base.cuh"

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
int fixed_base(const uint32_t* scalars_std, uint32_t n, uint32_t* out_std) {
  std::vector<Fr> s(n);
  std::vector<F> out((size_t)3 * n);
  std::memcpy(s.data(), scalars_std, (size_t)n * sizeof(Fr));
  int err = 0;
  if (fixed_base_mul<F>(s.data(), n, out.data(), &err, nullptr)) return 1;
  std::memcpy(out_std, out.data(), out.size() * sizeof(F));
  return err ? 100 + err : 0;
}
}  // namespace

extern "C" {
int t_fixed_base_c() { return kFixedBaseC; }
// out = n points (x, y, 1) standard form, infinity all zero; group 1 = G1, 2 = G2
int t_fixed_base(int group, const uint32_t* scalars_std, uint32_t n, uint32_t* out_std) {
  return group == 1 ? fixed_base<Fq>(scalars_std, n, out_std) : fixed_base<Fq2>(scalars_std, n, out_std);
}
}
