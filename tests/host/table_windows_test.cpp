// CPU test vehicle for MSMs over reduced window tables (B200_CFG_TABLE_WINDOWS; g++, csrc/host_stub): the library's own
// table build (window_table_enqueue) with t rows and its MSM engine (msm_host.cuh: grouped digit recode and counting
// sort over G*2^(c-1) buckets, both accumulation kernels, the slice merge, and the grouped tails — rows / columns and bit
// planes per window group with blockIdx.y = group, one Horner chain over all groups; or, for c < 7, scaled segment sums
// and a tree sum).  Reuses the CTA emulation of host_kernel_test.cpp.
// Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"

namespace {
template <class F>
int msm_grouped(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t t, uint32_t S,
                uint32_t* out_std) {
  if (t == 0 || t > (255 + c - 1) / c) return 98;
  int err = 0;
  Bases b;
  int rc = make_bases<F>(b, group, jac_std, n, c, t, S, &err);
  if (rc) return rc;
  std::vector<Fr> scalars(n);
  std::memcpy(scalars.data(), scalars_std, (size_t)n * sizeof(Fr));
  XYZZ<F> rec;
  if (msm_enqueue<F>(test_env(0), &b, scalars.data(), n, 0, &rec, &err, nullptr)) return 95;
  if (err) return 100 + err;
  if ((rc = check_sort(b.sort, b.sh))) return rc;
  finalize_std<F>(rec, out_std);
  return 0;
}

// k_tail_horner alone: planes_std holds groups * (nplanes + 1) affine points (x, y standard form)
template <class F>
int tail_horner(const uint32_t* planes_std, uint32_t nplanes, uint32_t groups, uint32_t gshift, uint32_t* out_std) {
  constexpr int W = sizeof(F) / 4;
  const size_t np = (size_t)groups * (nplanes + 1);
  std::vector<XYZZ<F>> planes(np);
  for (size_t i = 0; i < np; i++) {
    Affine<F> a{load_std<F>(planes_std + i * 2 * W), load_std<F>(planes_std + i * 2 * W + W)};
    planes[i] = XYZZ<F>::from_affine(a);
  }
  XYZZ<F> total_pt;
  run_cta(0, 32, 1, [&] { k_tail_horner<F>(planes.data(), nplanes, &total_pt, groups, gshift); });
  finalize_std<F>(total_pt, out_std);
  return 0;
}
}  // namespace

extern "C" {
// sum_i scalars[i] * P_i with a table of t window rows; S = 0: XYZZ accumulation, else batched-affine slices of S
int t_msm_grouped(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t t,
                  uint32_t S, uint32_t* out_std) {
  return group == 1 ? msm_grouped<Fq>(group, jac_std, scalars_std, n, c, t, S, out_std)
                    : msm_grouped<Fq2>(group, jac_std, scalars_std, n, c, t, S, out_std);
}
int t_tail_horner(int group, const uint32_t* planes_std, uint32_t nplanes, uint32_t groups, uint32_t gshift, uint32_t* out_std) {
  return group == 1 ? tail_horner<Fq>(planes_std, nplanes, groups, gshift, out_std)
                    : tail_horner<Fq2>(planes_std, nplanes, groups, gshift, out_std);
}
}
