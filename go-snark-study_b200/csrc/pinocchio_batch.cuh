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

// ---- key shards (b200_pinocchio_prove_witness_batch_record_device, b200_pinocchio_finalize_records_batch_device) -------
// Record of one rank for one proof: eight XYZZ slots of 256 B (0 PiA, 1 PiAp, 2 PiBp, 3 PiC, 4 PiCp, 5 PiH, 6 PiKp, 7 PiB
// in G2), 2 KB; a slot the rank does not own is infinity.
constexpr size_t kPinRecordBytes = 8 * 256;

// Thread e of 8k: slot s = e / k of proof p = e mod k from the batched MSMs' records (g1 as in k_pinocchio_finalize_batch,
// g2 the k PiB records) into record p at recs + 2 KB * p.  The caller zeroes the records first.
__global__ void k_pinocchio_records_batch(const XYZZ<Fq>* __restrict__ g1, const XYZZ<Fq2>* __restrict__ g2, uint32_t k,
                                          uint8_t* __restrict__ recs) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 8 * k) return;
  const uint32_t s = e / k, p = e - s * k;
  uint8_t* r = recs + kPinRecordBytes * (size_t)p + 256 * s;
  if (s < 7) *reinterpret_cast<XYZZ<Fq>*>(r) = g1[e];
  else *reinterpret_cast<XYZZ<Fq2>*>(r) = g2[p];
}

// world x k records -> k proofs.  The record of rank g for proof p is at recs + 2 KB * (g*k + p): the layout an all-gather
// of k records per rank leaves.  Proof p at out + 27p (F_q elements: 108 u64), the seven G1 points in slot order and then
// PiB, Jacobian, standard form; each point is infinity plus the ranks' records in rank order.  The 7k G1 sums take the
// first ceil(7k / 64) blocks and the k G2 sums blocks of their own; one proof (k = 1) is two blocks.
__global__ void k_pinocchio_gather_finalize_batch(const uint8_t* __restrict__ recs, int world, uint32_t k, Fq* __restrict__ out) {
  const uint32_t nb1 = (7 * k + kPinFinalizeBlock - 1) / kPinFinalizeBlock;
  const size_t rank_stride = kPinRecordBytes * (size_t)k;
  if (blockIdx.x < nb1) {
    const uint32_t e = blockIdx.x * kPinFinalizeBlock + threadIdx.x;
    if (e >= 7 * k) return;
    const uint32_t s = e / k, p = e - s * k;
    const uint8_t* r = recs + kPinRecordBytes * (size_t)p + 256 * s;
    XYZZ<Fq> acc = XYZZ<Fq>::inf();
    for (int g = 0; g < world; g++, r += rank_stride) xyzz_add(acc, *reinterpret_cast<const XYZZ<Fq>*>(r));
    store_jacobian_std(acc, out + 27 * (size_t)p + 3 * s);
  } else {
    const uint32_t p = (blockIdx.x - nb1) * kPinFinalizeBlock + threadIdx.x;
    if (p >= k) return;
    const uint8_t* r = recs + kPinRecordBytes * (size_t)p + 256 * 7;
    XYZZ<Fq2> acc = XYZZ<Fq2>::inf();
    for (int g = 0; g < world; g++, r += rank_stride) xyzz_add(acc, *reinterpret_cast<const XYZZ<Fq2>*>(r));
    store_jacobian_std(acc, reinterpret_cast<Fq2*>(out + 27 * (size_t)p + 21));
  }
}
inline unsigned pinocchio_finalize_blocks(uint32_t k) {
  return (7 * k + kPinFinalizeBlock - 1) / kPinFinalizeBlock + (k + kPinFinalizeBlock - 1) / kPinFinalizeBlock;
}

}  // namespace b200
