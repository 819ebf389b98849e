// The partial records of Groth16 proofs on a key shard and their finalisation, for one proof and for batches of k
// (b200_groth16_prove_witness_batch_partial_device, b200_groth16_finalize_batch_device).  In a header of its own so that
// the CPU test vehicle (tests/host/shard_batch_test.cpp) runs the kernels the library launches.
#pragma once
#include "ec.cuh"

namespace b200 {

// Partial record of one rank for one proof: A (G1 XYZZ @ +0), B1 (@ +256), B2 (G2 XYZZ @ +512), C part with the rank's
// blinding products folded in (@ +768) — 1 KB.
constexpr size_t kPartialBytes = 1024;
constexpr uint32_t kG16FinalizeBlock = 32;

// Thread p of a batch: record p at recs + 1 KB * p from the batched MSMs' k records per set, CH_p + prod[2p] + prod[2p+1]
// in the C slot (the additions of k_groth16_fold_products, in its order).  The caller zeroes the records first, so the
// bytes between the slots are zero.
__global__ void k_groth16_fold_products_batch(const XYZZ<Fq>* __restrict__ rA, const XYZZ<Fq>* __restrict__ rB1,
                                              const XYZZ<Fq2>* __restrict__ rB2, const XYZZ<Fq>* __restrict__ rCH,
                                              const XYZZ<Fq>* __restrict__ prod, uint32_t k, uint8_t* __restrict__ recs) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= k) return;
  uint8_t* rec = recs + kPartialBytes * (size_t)p;
  XYZZ<Fq> c = rCH[p];
  xyzz_add(c, prod[2 * p]);
  xyzz_add(c, prod[2 * p + 1]);
  *reinterpret_cast<XYZZ<Fq>*>(rec) = rA[p];
  *reinterpret_cast<XYZZ<Fq>*>(rec + 256) = rB1[p];
  *reinterpret_cast<XYZZ<Fq2>*>(rec + 512) = rB2[p];
  *reinterpret_cast<XYZZ<Fq>*>(rec + 768) = c;
}

// world x k partial records -> k proofs.  The record of rank g for proof p is at parts + 1 KB * (g*k + p): the layout an
// all-gather of k records per rank leaves.  Proof p at out + 12p (F_q elements: 48 u64), PiA | PiC | PiB, Jacobian,
// standard form.  Each point is rank 0's record plus ranks 1 .. world-1 in order.  Blocks [0, nb) sum PiA, [nb, 2nb) PiC
// and [2nb, 3nb) PiB (nb = ceil(k / 32)), so no warp runs both field towers; one proof (k = 1) is three blocks.
__global__ void k_groth16_finalize_batch(const uint8_t* __restrict__ parts, int world, uint32_t k, Fq* __restrict__ out) {
  const uint32_t nb = (k + kG16FinalizeBlock - 1) / kG16FinalizeBlock;
  const uint32_t j = blockIdx.x / nb, p = (blockIdx.x - j * nb) * kG16FinalizeBlock + threadIdx.x;
  if (p >= k) return;
  const size_t rank_stride = kPartialBytes * (size_t)k;
  const uint8_t* rec = parts + kPartialBytes * (size_t)p + (j == 0 ? 0 : j == 1 ? 768 : 512);
  Fq* o = out + 12 * (size_t)p + 3 * j;
  if (j < 2) {
    XYZZ<Fq> acc = *reinterpret_cast<const XYZZ<Fq>*>(rec);
    for (int g = 1; g < world; g++) {
      rec += rank_stride;
      xyzz_add(acc, *reinterpret_cast<const XYZZ<Fq>*>(rec));
    }
    store_jacobian_std(acc, o);
  } else {
    XYZZ<Fq2> acc = *reinterpret_cast<const XYZZ<Fq2>*>(rec);
    for (int g = 1; g < world; g++) {
      rec += rank_stride;
      xyzz_add(acc, *reinterpret_cast<const XYZZ<Fq2>*>(rec));
    }
    store_jacobian_std(acc, reinterpret_cast<Fq2*>(o));
  }
}

inline unsigned groth16_finalize_blocks(uint32_t k) { return 3 * ((k + kG16FinalizeBlock - 1) / kG16FinalizeBlock); }

}  // namespace b200
