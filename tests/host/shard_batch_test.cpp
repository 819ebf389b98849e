// CPU test vehicle for the kernels of batched proving on key shards (g++, csrc/host_stub): the finalisation of world x k
// Groth16 partial records (k_groth16_finalize_batch), the quotient store of a shard's C||PTD vectors (k_quotient_store
// with a source offset) and the gather-finalisation of world x k Pinocchio records (k_pinocchio_gather_finalize_batch), each run one emulated thread at a time with the launch shape the library uses.
// Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"
#include "shard_batch.cuh"
#include "pinocchio_batch.cuh"

namespace {
template <class F>
XYZZ<F> xyzz_of(const uint32_t* xy, const uint32_t* u_std) {   // affine (standard form; (0, 0) is infinity) scaled by u
  constexpr int W = sizeof(F) / 4;
  Affine<F> a{load_std<F>(xy), load_std<F>(xy + W)};
  F u = load_std<F>(u_std), u2 = u.sqr(), u3 = u2 * u;
  return a.is_inf() ? XYZZ<F>::inf() : XYZZ<F>{a.x * u2, a.y * u3, u2, u3};
}
}  // namespace

extern "C" {
// Records from affine points: record e = g*k + p (rank g, proof p) holds A, B1, C from g1_xy[3e .. 3e+2] (2 F_q each)
// and B2 from g2_xy[e] (2 F_q2), each XYZZ with ZZ = u^2, ZZZ = u^3 for its scale (3 world k F_q, then world k F_q2).
// out_batch: k_groth16_finalize_batch over all records (k x 12 F_q); out_single: per proof p, the kernel with k = 1 over
// that proof's world records copied out contiguously (the single proof's finalisation), at out_single + 12p F_q.
int t_groth16_finalize_batch(const uint32_t* g1_xy, const uint32_t* g2_xy, const uint32_t* scale, int world, uint32_t k,
                             uint32_t* out_batch, uint32_t* out_single) {
  const size_t nrec = (size_t)world * k;
  std::vector<uint8_t> recs(nrec * kPartialBytes, 0xa5);   // the bytes between the slots are never read
  for (size_t e = 0; e < nrec; e++) {
    uint8_t* r = recs.data() + kPartialBytes * e;
    const size_t offs[3] = {0, 256, 768};
    for (int j = 0; j < 3; j++)
      *reinterpret_cast<XYZZ<Fq>*>(r + offs[j]) = xyzz_of<Fq>(g1_xy + 16 * (3 * e + j), scale + 8 * (3 * e + j));
    *reinterpret_cast<XYZZ<Fq2>*>(r + 512) = xyzz_of<Fq2>(g2_xy + 32 * e, scale + 8 * 3 * nrec + 16 * e);
  }
  std::vector<Fq> o(12 * (size_t)k);
  for (auto& v : o) v.l[0] = 0xdeadbeefu;
  run_threads(groth16_finalize_blocks(k), kG16FinalizeBlock, [&] { k_groth16_finalize_batch(recs.data(), world, k, o.data()); });
  std::memcpy(out_batch, o.data(), o.size() * sizeof(Fq));
  std::vector<uint8_t> one((size_t)world * kPartialBytes);
  for (uint32_t p = 0; p < k; p++) {
    for (int g = 0; g < world; g++)
      std::memcpy(one.data() + kPartialBytes * g, recs.data() + kPartialBytes * ((size_t)g * k + p), kPartialBytes);
    Fq o1[12];
    run_threads(groth16_finalize_blocks(1), kG16FinalizeBlock, [&] { k_groth16_finalize_batch(one.data(), world, 1, o1); });
    std::memcpy(out_single + 96 * (size_t)p, o1, sizeof o1);
  }
  return 0;
}

// k_quotient_store over k vectors of `stride` scalars (standard form, in place) from scalar `base` of each (a shard's
// C||PTD vectors from their PowersTauDelta slice): coef_std as t_quotient_store of prove_batch_test.cpp (k blocks of
// cstride, standard form; null: the entries in place stay), off = the slice's first quotient index, nslot its length,
// tail_std: k scalars (-r_p s_p) or null (the shard does not hold the tail).
int t_quotient_store_shard(const uint32_t* coef_std, uint32_t cstride, uint32_t nh, uint32_t off, uint32_t nslot,
                           const uint32_t* tail_std, uint32_t k, uint32_t stride, uint32_t base, uint32_t* vec_std) {
  std::vector<Fr> coef(coef_std ? (size_t)k * cstride : 0), tail(tail_std ? k : 0), vec((size_t)k * stride);
  for (size_t i = 0; i < coef.size(); i++) coef[i] = load_std<Fr>(coef_std + 8 * i);   // Montgomery, as the front end leaves it
  if (tail_std) std::memcpy(tail.data(), tail_std, tail.size() * sizeof(Fr));   // standard form, as the library's
  std::memcpy(vec.data(), vec_std, vec.size() * sizeof(Fr));
  const uint32_t total = k * (nslot + 1);
  run_threads(cdiv(total, 256), 256, [&] {
    k_quotient_store(coef_std ? coef.data() : nullptr, cstride, nh, nslot, tail_std ? tail.data() : nullptr, 1, total,
                     vec.data() + base, stride, off);
  });
  std::memcpy(vec_std, vec.data(), vec.size() * sizeof(Fr));
  return 0;
}
// Pinocchio records from affine points: record e = g*k + p holds its seven G1 slots from g1_xy[7e .. 7e+6] and PiB from
// g2_xy[e], scaled as in t_groth16_finalize_batch (7 world k F_q, then world k F_q2).  out_batch: the batch kernel (k x 27
// F_q); out_single: per proof p, the kernel with k = 1 over that proof's world records copied out contiguously (the
// single proof's gather-finalisation), at out_single + 27p F_q.
int t_pinocchio_gather_finalize_batch(const uint32_t* g1_xy, const uint32_t* g2_xy, const uint32_t* scale, int world,
                                      uint32_t k, uint32_t* out_batch, uint32_t* out_single) {
  const size_t nrec = (size_t)world * k;
  std::vector<uint8_t> recs(nrec * kPinRecordBytes, 0xa5);
  for (size_t e = 0; e < nrec; e++) {
    uint8_t* r = recs.data() + kPinRecordBytes * e;
    for (int s = 0; s < 7; s++)
      *reinterpret_cast<XYZZ<Fq>*>(r + 256 * s) = xyzz_of<Fq>(g1_xy + 16 * (7 * e + s), scale + 8 * (7 * e + s));
    *reinterpret_cast<XYZZ<Fq2>*>(r + 256 * 7) = xyzz_of<Fq2>(g2_xy + 32 * e, scale + 8 * 7 * nrec + 16 * e);
  }
  std::vector<Fq> o(27 * (size_t)k);
  for (auto& v : o) v.l[0] = 0xdeadbeefu;
  run_threads(pinocchio_finalize_blocks(k), kPinFinalizeBlock, [&] { k_pinocchio_gather_finalize_batch(recs.data(), world, k, o.data()); });
  std::memcpy(out_batch, o.data(), o.size() * sizeof(Fq));
  std::vector<uint8_t> one((size_t)world * kPinRecordBytes);
  for (uint32_t p = 0; p < k; p++) {
    for (int g = 0; g < world; g++)
      std::memcpy(one.data() + kPinRecordBytes * g, recs.data() + kPinRecordBytes * ((size_t)g * k + p), kPinRecordBytes);
    Fq o1[27];
    run_threads(pinocchio_finalize_blocks(1), kPinFinalizeBlock, [&] { k_pinocchio_gather_finalize_batch(one.data(), world, 1, o1); });
    std::memcpy(out_single + 216 * (size_t)p, o1, sizeof o1);
  }
  return 0;
}
}
