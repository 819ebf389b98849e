// CPU test vehicle for MSMs over reduced window tables (B200_CFG_TABLE_WINDOWS; g++, csrc/host_stub): the library's own
// table build (window_table_enqueue) with t rows, the grouped digit recode and counting sort over G*2^(c-1) buckets, both
// accumulation kernels, the slice merge, and the grouped tails (rows / columns and bit planes per window group with
// blockIdx.y = group, one Horner chain over all groups; or, for c < 7, scaled segment sums and a tree sum), kernel by
// kernel in the order capi.cu issues them.  Reuses the CTA emulation of host_kernel_test.cpp.
// Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"
#include "fixed_base.cuh"

namespace {
// run `kernel` as window group g of a 2-D grid (blockIdx.y = g in every emulated thread)
template <class K>
void run_cta_group(unsigned b, unsigned g, unsigned nthreads, unsigned nblocks, K kernel) {
  run_cta(b, nthreads, nblocks, [&, g] {
    blockIdx.y = g;
    kernel();
  });
}

template <class F>
int msm_grouped(const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t t, uint32_t S,
                uint32_t* out_std) {
  MsmShape sh{n, c, (255 + c - 1) / c, 1u << (c - 1), n};
  if (t == 0 || t > sh.nwin) return 98;
  sh.rows = t;
  sh.groups = (sh.nwin + t - 1) / t;
  const uint32_t B = total_buckets(sh), G = sh.groups, gshift = c * t;
  int err = 0;
  // --- bases_create: t table rows
  std::vector<F> staging((size_t)n * 3);
  std::memcpy(staging.data(), jac_std, staging.size() * sizeof(F));
  std::vector<Affine<F>> table((size_t)t * n);
  std::vector<XYZZ<F>> state(n);
  window_table_enqueue<F>(staging.data(), n, t, (int)c, table.data(), state.data(), &err, nullptr);
  // --- msm_sort over G*2^(c-1) buckets
  uint32_t m = B + 1;
  uint64_t total = (uint64_t)sh.nwin * n;
  uint64_t mean = (total + B - 1) / B;
  uint32_t cap = (uint32_t)(2 * mean < 32 ? 32 : 2 * mean);
  int fixed = 0;
  if (S) {
    cap = S;
    fixed = 1;
  }
  size_t max_slices = B + total / (S ? S : cap) + 8 + (S ? 0 : B);
  std::vector<Fr> scalars(n);
  std::memcpy(scalars.data(), scalars_std, (size_t)n * sizeof(Fr));
  std::vector<uint32_t> counts(m + 1, 0), offsets(m + 1, 0), cursor(m + 1, 0), entries(total + 8, 0);
  std::vector<uint32_t> slice_off(m + 2, 0), slice_start(max_slices, 0), slice_end(max_slices, 0);
  SliceTables stb{slice_off.data(), slice_start.data(), slice_end.data()};
  run_threads(cdiv(n, 256), 256, [&] { k_digits_count(scalars.data(), sh, 0, counts.data(), &err); });
  run_cta(0, 256, 1, [&] { k_scan(counts.data(), m, cap, fixed, offsets.data(), cursor.data(), stb); });
  run_threads(cdiv(m, 256), 256, [&] { k_fill_slices(counts.data(), offsets.data(), m, cap, fixed, stb); });
  run_threads(cdiv(n, 256), 256, [&] { k_digits_scatter(scalars.data(), sh, 0, cursor.data(), entries.data(), &err); });
  if (err) return 100 + err;
  for (uint32_t k = 0; k < offsets[m]; k++)
    if ((entries[k] >> 1) >= (size_t)t * n) return 96;   // every entry reads one of the t stored rows
  uint32_t nslices = slice_off[m];
  if (nslices > max_slices) return 99;
  // --- msm_buckets
  std::vector<XYZZ<F>> buckets(B);
  if (S) {
    uint32_t R = 0;
    while ((1u << R) < S) R++;
    constexpr int T = 8;
    const size_t capn = (size_t)nslices * (S / 2) + 1;
    std::vector<F> bufA(2 * capn), bufB(2 * capn);
    std::vector<F> pre(capn);
    std::vector<uint2> ids(capn);
    unsigned nb_max = cdiv((size_t)nslices * (S / 2), kAffBlock * T) + 1;
    std::vector<F> others((size_t)nb_max * kAffBlock), btot(nb_max);
    AffineRound<F> ar{};
    ar.table = table.data();
    ar.entries = entries.data();
    ar.slice_start = slice_start.data();
    ar.slice_end = slice_end.data();
    ar.nslices_ptr = slice_off.data() + m;
    ar.pre = pre.data();
    ar.others = others.data();
    ar.btot = btot.data();
    ar.pair_ids = ids.data();
    NodeBuf<F> prev{nullptr, nullptr};
    NodeBuf<F> bufs[2] = {{bufA.data(), bufA.data() + capn}, {bufB.data(), bufB.data() + capn}};
    for (uint32_t r = 1; r <= R; r++) {
      ar.round = r;
      ar.q_log = R - r;
      ar.prev = prev;
      ar.out = bufs[(r - 1) & 1];
      unsigned nb = cdiv((size_t)nslices << ar.q_log, kAffBlock * T);
      if (nb == 0) nb = 1;
      for (unsigned b = 0; b < nb; b++) run_cta(b, kAffBlock, nb, [&] { k_affine_forward<F, T, 1>(ar); });
      for (unsigned b = 0; b < cdiv((size_t)nb * 32, 128); b++) run_cta(b, 128, cdiv((size_t)nb * 32, 128), [&] { k_affine_invert<F>(ar.btot, nb); });
      run_backward<F, T>(0, ar, nb);
      prev = ar.out;
    }
    for (unsigned b = 0; b < cdiv(B, 128); b++)
      run_cta(b, 128, cdiv(B, 128), [&] { k_merge_slices_affine<F>(prev, stb, B, buckets.data()); });
  } else {
    std::vector<XYZZ<F>> slice_out(max_slices);
    unsigned nb = cdiv((size_t)max_slices * 2, 128);
    for (unsigned b = 0; b < nb; b++) run_cta(b, 128, nb, [&] { k_accumulate<F, 2>(table.data(), entries.data(), stb, m, slice_out.data()); });
    for (unsigned b = 0; b < cdiv(B, 128); b++)
      run_cta(b, 128, cdiv(B, 128), [&] { k_merge_slices<F>(slice_out.data(), stb, B, buckets.data()); });
  }
  // --- the grouped tail
  XYZZ<F> total_pt;
  if (c >= 7) {
    const uint32_t bits = c - 1, kl = (bits + 1) / 2, kh = bits - kl, K = 1u << kl, H = 1u << kh;
    std::vector<XYZZ<F>> scratch((size_t)G * (H + K + bits + 1));
    XYZZ<F>*Rr = scratch.data(), *Cc = Rr + (size_t)G * H, *planes = Cc + (size_t)G * K;
    unsigned nb1 = cdiv((size_t)(H + K) * 32, 128), nb2 = cdiv((size_t)(bits + 1) * 32, 128);
    for (unsigned g = 0; g < G; g++)
      for (unsigned b = 0; b < nb1; b++) run_cta_group(b, g, 128, nb1, [&] { k_tail_rowcol<F>(buckets.data(), kl, H, Rr, Cc); });
    for (unsigned g = 0; g < G; g++)
      for (unsigned b = 0; b < nb2; b++) run_cta_group(b, g, 128, nb2, [&] { k_tail_planes<F>(Rr, Cc, kl, kh, planes); });
    run_cta(0, 32, 1, [&] { k_tail_horner<F>(planes, bits, &total_pt, G, gshift); });
  } else {
    uint32_t seg = sh.nbuckets >= 256 ? 4 : 1, nseg = (sh.nbuckets + seg - 1) / seg;
    std::vector<XYZZ<F>> partials((size_t)G * nseg + 1024);
    for (unsigned g = 0; g < G; g++)
      for (unsigned b = 0; b < cdiv(nseg, 128); b++)
        run_cta_group(b, g, 128, cdiv(nseg, 128), [&] { k_bucket_reduce<F>(buckets.data(), sh.nbuckets, seg, partials.data(), nseg, gshift); });
    const uint32_t cnt = G * nseg;
    if (cnt <= 64) {
      run_cta(0, 256, 1, [&] { k_sum_points<F>(partials.data(), cnt, cnt, &total_pt); });
    } else {   // the two-level tree sum of launch_tree_sum, with a lower switch point so small inputs reach it
      uint32_t per = 32, nb2 = (cnt + per - 1) / per;
      for (unsigned b = 0; b < nb2; b++) run_cta(b, 256, nb2, [&] { k_sum_points<F>(partials.data(), cnt, per, partials.data() + cnt); });
      run_cta(0, 256, 1, [&] { k_sum_points<F>(partials.data() + cnt, nb2, nb2, &total_pt); });
    }
  }
  F out[3];
  run_cta(0, 32, 1, [&] { k_finalize<F>(&total_pt, out); });
  std::memcpy(out_std, out, sizeof out);
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
  F out[3];
  run_cta(0, 32, 1, [&] { k_finalize<F>(&total_pt, out); });
  std::memcpy(out_std, out, sizeof out);
  return 0;
}
}  // namespace

extern "C" {
// sum_i scalars[i] * P_i with a table of t window rows; S = 0: XYZZ accumulation, else batched-affine slices of S
int t_msm_grouped(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t t,
                  uint32_t S, uint32_t* out_std) {
  return group == 1 ? msm_grouped<Fq>(jac_std, scalars_std, n, c, t, S, out_std)
                    : msm_grouped<Fq2>(jac_std, scalars_std, n, c, t, S, out_std);
}
int t_tail_horner(int group, const uint32_t* planes_std, uint32_t nplanes, uint32_t groups, uint32_t gshift, uint32_t* out_std) {
  return group == 1 ? tail_horner<Fq>(planes_std, nplanes, groups, gshift, out_std)
                    : tail_horner<Fq2>(planes_std, nplanes, groups, gshift, out_std);
}
}
