// CPU test vehicle for the kernels of b200_pinocchio_prove_witness_batch (g++, csrc/host_stub): the quotient store into
// the G1T scalar vectors (k_quotient_store with no tail element) and the finalisation of the 8k XYZZ records
// (k_pinocchio_finalize_batch), each run one emulated thread at a time with the launch shape the library uses.
// Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"
#include "pinocchio_batch.cuh"

extern "C" {
// k quotients (coef_std: k blocks of cstride, standard form on input: converted to Montgomery here, so the kernel's
// conversion gives them back; null: the vectors' own entries below nh stay) -> vec_std: k vectors of n_g1t scalars.
int t_quotient_store_g1t(const uint32_t* coef_std, uint32_t cstride, uint32_t nh, uint32_t n_g1t, uint32_t k, uint32_t* vec_std) {
  std::vector<Fr> coef(coef_std ? (size_t)k * cstride : 0), vec((size_t)k * n_g1t);
  for (size_t i = 0; i < coef.size(); i++) coef[i] = load_std<Fr>(coef_std + 8 * i);
  std::memcpy(vec.data(), vec_std, vec.size() * sizeof(Fr));
  const uint32_t total = k * (n_g1t + 1);
  run_threads(cdiv(total, 256), 256, [&] {
    k_quotient_store(coef_std ? coef.data() : nullptr, cstride, nh, n_g1t, nullptr, 0, total, vec.data(), n_g1t);
  });
  std::memcpy(vec_std, vec.data(), vec.size() * sizeof(Fr));
  return 0;
}

// Records from affine points (standard form; (0, 0) is infinity): record e becomes the XYZZ point (x u^2, y u^3, u^2, u^3)
// with u = scale[e] (7k F_q, then k F_q2 elements), so the kernel's Jacobian output has Z = u^3 != 1.  g1_xy: 7k points
// of 2 F_q, slot-major (g1_xy[s*k + p]); g2_xy: k points of 2 F_q2; out: k x 27 F_q (216 u32 per proof).
int t_pinocchio_finalize_batch(const uint32_t* g1_xy, const uint32_t* g2_xy, const uint32_t* scale, uint32_t k, uint32_t* out) {
  std::vector<XYZZ<Fq>> r1(7 * (size_t)k);
  std::vector<XYZZ<Fq2>> r2(k);
  for (size_t e = 0; e < r1.size(); e++) {
    Affine<Fq> a{load_std<Fq>(g1_xy + 16 * e), load_std<Fq>(g1_xy + 16 * e + 8)};
    Fq u = load_std<Fq>(scale + 8 * e), u2 = u.sqr(), u3 = u2 * u;
    r1[e] = a.is_inf() ? XYZZ<Fq>::inf() : XYZZ<Fq>{a.x * u2, a.y * u3, u2, u3};
  }
  for (size_t p = 0; p < k; p++) {
    Affine<Fq2> a{load_std<Fq2>(g2_xy + 32 * p), load_std<Fq2>(g2_xy + 32 * p + 16)};
    Fq2 v = load_std<Fq2>(scale + 8 * 7 * (size_t)k + 16 * p), v2 = v.sqr(), v3 = v2 * v;
    r2[p] = a.is_inf() ? XYZZ<Fq2>::inf() : XYZZ<Fq2>{a.x * v2, a.y * v3, v2, v3};
  }
  std::vector<Fq> o(27 * (size_t)k);
  for (auto& v : o) v.l[0] = 0xdeadbeefu;
  run_threads(cdiv(7 * k, kPinFinalizeBlock) + cdiv(k, kPinFinalizeBlock), kPinFinalizeBlock,
              [&] { k_pinocchio_finalize_batch(r1.data(), r2.data(), k, o.data()); });
  std::memcpy(out, o.data(), o.size() * sizeof(Fq));
  return 0;
}
}
