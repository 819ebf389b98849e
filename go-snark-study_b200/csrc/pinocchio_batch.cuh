// The finalisation kernel of a batch of Pinocchio proofs (b200_pinocchio_prove_witness_batch): the batched MSMs' XYZZ
// records -> k proofs in standard form.  In a header of its own so that the CPU test vehicle
// (tests/host/pinocchio_batch_test.cpp) runs the kernel the library launches.
#pragma once
#include "ec.cuh"

namespace b200 {

constexpr uint32_t kPinFinalizeBlock = 64;
// One thread per record.  g1: 7 x k records, record p of result slot s (0 PiA, 1 PiAp, 2 PiBp, 3 PiC, 4 PiCp, 5 PiH,
// 6 PiKp) at g1[s*k + p]; g2: the k PiB records.  Proof p at out + 27p (F_q elements: 108 u64), its seven G1 points in
// slot order and then PiB.  The G1 records take the first ceil(7k / 64) blocks and the G2 records blocks of their own, so
// no warp runs both field towers.
__global__ void k_pinocchio_finalize_batch(const XYZZ<Fq>* __restrict__ g1, const XYZZ<Fq2>* __restrict__ g2, uint32_t k,
                                           Fq* __restrict__ out) {
  const uint32_t nb1 = (7 * k + kPinFinalizeBlock - 1) / kPinFinalizeBlock;
  if (blockIdx.x < nb1) {
    const uint32_t e = blockIdx.x * kPinFinalizeBlock + threadIdx.x;
    if (e >= 7 * k) return;
    const uint32_t s = e / k, p = e - s * k;
    store_jacobian_std(g1[e], out + 27 * (size_t)p + 3 * s);
  } else {
    const uint32_t p = (blockIdx.x - nb1) * kPinFinalizeBlock + threadIdx.x;
    if (p >= k) return;
    store_jacobian_std(g2[p], reinterpret_cast<Fq2*>(out + 27 * (size_t)p + 21));
  }
}

}  // namespace b200
