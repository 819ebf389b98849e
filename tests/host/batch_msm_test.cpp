// CPU test vehicle for batches of MSMs over one base set (b200_msm_device_batch; g++, csrc/host_stub): k scalar vectors
// through the batched digit recode and counting sort (vector p's digits in window groups p*G .. p*G + G - 1), the
// multi-block counter scan, both accumulation kernels, the slice merge, and the per-vector tails (rows / columns and bit
// planes over (vector, group) as blockIdx.y, one Horner chain per vector as blockIdx.x; or, for c < 7, scaled segment
// sums and one tree-sum block per vector), kernel by kernel in the order capi.cu issues them.  With `single` set, the
// same inputs also run the one-MSM sequence (one scan block, tree sum, one Horner block) so that k = 1 can be compared
// with it array by array.  Reuses the CTA emulation of host_kernel_test.cpp and the table build of fixed_base.cuh.
// Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"
#include "fixed_base.cuh"

namespace {
template <class K>
void run_cta_y(unsigned b, unsigned y, unsigned nthreads, unsigned nblocks, K kernel) {
  run_cta(b, nthreads, nblocks, [&, y] {
    blockIdx.y = y;
    kernel();
  });
}

// Everything a run leaves behind, for the k = 1 comparison.
template <class F>
struct BatchRun {
  std::vector<uint32_t> offsets, slice_off, slice_start, slice_end, entries;
  std::vector<XYZZ<F>> buckets, records;
};

// k vectors of n scalars (vector p at scalars + p*stride) over a table of t rows; scan_chunk > 0: the counter scan in
// blocks of scan_chunk counters (k_scan_totals + k_scan), else one block; single: the one-MSM launch sequence (k = 1).
// The (vector, group) tail kernels run in for_each_tail_chunk's chunks of at most max_rows rows, with the pointer offsets
// capi.cu gives each chunk (65535 on the device; a small max_rows puts chunk boundaries inside a batch).
template <class F>
int msm_batch(const std::vector<Affine<F>>& table, const Fr* scalars, uint32_t n, uint32_t k, uint32_t stride, uint32_t c,
              uint32_t t, uint32_t S, uint32_t scan_chunk, bool single, BatchRun<F>& run, uint32_t max_rows = 65535) {
  MsmShape sh{n, c, (255 + c - 1) / c, 1u << (c - 1), n};
  sh.rows = t;
  sh.groups = (sh.nwin + t - 1) / t;
  sh.vecs = k;
  sh.vec_stride = stride;
  const uint32_t B = total_buckets(sh), G = sh.groups, gshift = c * t, m = B + 1;
  int err = 0;
  // --- msm_sort over k*G*2^(c-1) buckets; the slice cap is that of one vector
  const uint64_t total = (uint64_t)k * sh.nwin * n;
  const uint64_t mean = (total + B - 1) / B;
  uint32_t cap = (uint32_t)(2 * mean < 32 ? 32 : 2 * mean);
  int fixed = 0;
  if (S) {
    cap = S;
    fixed = 1;
  }
  const size_t max_slices = B + total / (S ? S : cap) + 8 + (S ? 0 : B);
  std::vector<uint32_t> counts(m + 1, 0), cursor(m + 1, 0);
  run.offsets.assign(m + 1, 0);
  run.entries.assign(total + 8, 0);
  run.slice_off.assign(m + 2, 0);
  run.slice_start.assign(max_slices, 0);
  run.slice_end.assign(max_slices, 0);
  SliceTables stb{run.slice_off.data(), run.slice_start.data(), run.slice_end.data()};
  const size_t nterm = (size_t)k * n;
  run_threads(cdiv(nterm, 256), 256, [&] { k_digits_count(scalars, sh, 0, counts.data(), &err); });
  if (scan_chunk) {
    const unsigned nb = cdiv(m, scan_chunk);
    std::vector<unsigned long long> totals(nb);
    for (unsigned b = 0; b < nb; b++) run_cta(b, 256, nb, [&] { k_scan_totals(counts.data(), m, cap, scan_chunk, totals.data()); });
    for (unsigned b = 0; b < nb; b++)
      run_cta(b, 256, nb, [&] { k_scan(counts.data(), m, cap, fixed, run.offsets.data(), cursor.data(), stb, scan_chunk, totals.data()); });
  } else {
    run_cta(0, 256, 1, [&] { k_scan(counts.data(), m, cap, fixed, run.offsets.data(), cursor.data(), stb); });
  }
  run_threads(cdiv(m, 256), 256, [&] { k_fill_slices(counts.data(), run.offsets.data(), m, cap, fixed, stb); });
  run_threads(cdiv(nterm, 256), 256, [&] { k_digits_scatter(scalars, sh, 0, cursor.data(), run.entries.data(), &err); });
  if (err) return 100 + err;
  for (uint32_t e = 0; e < run.offsets[m]; e++)
    if ((run.entries[e] >> 1) >= (size_t)t * n) return 96;   // every entry reads one of the t stored rows of base < n
  for (uint32_t b = 1; b < m; b++)
    if (cursor[b] != run.offsets[b + 1]) return 97;          // each bucket filled exactly to the next one's offset
  const uint32_t nslices = run.slice_off[m];
  if (nslices > max_slices) return 99;
  // --- bucket_phase
  run.buckets.assign(B, XYZZ<F>{});
  XYZZ<F>* buckets = run.buckets.data();
  if (S) {
    uint32_t R = 0;
    while ((1u << R) < S) R++;
    constexpr int T = 8;
    const size_t capn = (size_t)nslices * (S / 2) + 1;
    std::vector<F> bufA(2 * capn), bufB(2 * capn), pre(capn);
    std::vector<uint2> ids(capn);
    unsigned nb_max = cdiv((size_t)nslices * (S / 2), kAffBlock * T) + 1;
    std::vector<F> others((size_t)nb_max * kAffBlock), btot(nb_max);
    AffineRound<F> ar{};
    ar.table = table.data();
    ar.entries = run.entries.data();
    ar.slice_start = run.slice_start.data();
    ar.slice_end = run.slice_end.data();
    ar.nslices_ptr = run.slice_off.data() + m;
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
    for (unsigned b = 0; b < cdiv(B, 128); b++) run_cta(b, 128, cdiv(B, 128), [&] { k_merge_slices_affine<F>(prev, stb, B, buckets); });
  } else {
    std::vector<XYZZ<F>> slice_out(max_slices);
    unsigned nb = cdiv((size_t)max_slices * 2, 128);
    for (unsigned b = 0; b < nb; b++) run_cta(b, 128, nb, [&] { k_accumulate<F, 2>(table.data(), run.entries.data(), stb, m, slice_out.data()); });
    for (unsigned b = 0; b < cdiv(B, 128); b++) run_cta(b, 128, cdiv(B, 128), [&] { k_merge_slices<F>(slice_out.data(), stb, B, buckets); });
  }
  // --- the tails: one record per vector
  run.records.assign(k, XYZZ<F>{});
  const uint32_t GV = k * G;
  if (c >= 7) {
    const uint32_t bits = c - 1, kl = (bits + 1) / 2, kh = bits - kl, K = 1u << kl, H = 1u << kh;
    std::vector<XYZZ<F>> scratch((size_t)GV * (H + K + bits + 1));
    XYZZ<F>*Rr = scratch.data(), *Cc = Rr + (size_t)GV * H, *planes = Cc + (size_t)GV * K;
    unsigned nb1 = cdiv((size_t)(H + K) * 32, 128), nb2 = cdiv((size_t)(bits + 1) * 32, 128);
    for_each_tail_chunk(sh, max_rows, [&](uint32_t y0, uint32_t ny) {
      const XYZZ<F>* bk = buckets + (size_t)y0 * H * K;
      XYZZ<F>*r = Rr + (size_t)y0 * H, *cc = Cc + (size_t)y0 * K, *pl = planes + (size_t)y0 * (bits + 1);
      for (unsigned y = 0; y < ny; y++)
        for (unsigned b = 0; b < nb1; b++) run_cta_y(b, y, 128, nb1, [&] { k_tail_rowcol<F>(bk, kl, H, r, cc); });
      for (unsigned y = 0; y < ny; y++)
        for (unsigned b = 0; b < nb2; b++) run_cta_y(b, y, 128, nb2, [&] { k_tail_planes<F>(r, cc, kl, kh, pl); });
    });
    for (unsigned v = 0; v < k; v++) run_cta(v, 32, k, [&] { k_tail_horner<F>(planes, bits, run.records.data(), G, gshift); });
  } else {
    uint32_t seg = sh.nbuckets >= 256 ? 4 : 1, nseg = (sh.nbuckets + seg - 1) / seg;
    std::vector<XYZZ<F>> partials((size_t)GV * nseg + 1024);
    const uint32_t per = G * nseg;
    if (single) {   // launch_segment_tail for one vector: no group modulus, then launch_tree_sum (lower switch point)
      for (unsigned y = 0; y < G; y++)
        for (unsigned b = 0; b < cdiv(nseg, 128); b++)
          run_cta_y(b, y, 128, cdiv(nseg, 128), [&] { k_bucket_reduce<F>(buckets, sh.nbuckets, seg, partials.data(), nseg, gshift); });
      if (per <= 64) {
        run_cta(0, 256, 1, [&] { k_sum_points<F>(partials.data(), per, per, run.records.data()); });
      } else {
        uint32_t pb = 32, nb2 = (per + pb - 1) / pb;
        for (unsigned b = 0; b < nb2; b++) run_cta(b, 256, nb2, [&] { k_sum_points<F>(partials.data(), per, pb, partials.data() + per); });
        run_cta(0, 256, 1, [&] { k_sum_points<F>(partials.data() + per, nb2, nb2, run.records.data()); });
      }
    } else {
      for_each_tail_chunk(sh, max_rows, [&](uint32_t y0, uint32_t ny) {
        const XYZZ<F>* bk = buckets + (size_t)y0 * sh.nbuckets;
        XYZZ<F>* out = partials.data() + (size_t)y0 * nseg;
        for (unsigned y = 0; y < ny; y++)
          for (unsigned b = 0; b < cdiv(nseg, 128); b++)
            run_cta_y(b, y, 128, cdiv(nseg, 128), [&] { k_bucket_reduce<F, true>(bk, sh.nbuckets, seg, out, nseg, gshift, G); });
      });
      for (unsigned v = 0; v < k; v++) run_cta(v, 256, k, [&] { k_sum_points<F>(partials.data(), GV * nseg, per, run.records.data()); });
    }
  }
  return 0;
}

template <class F>
std::vector<Affine<F>> make_table(const uint32_t* jac_std, uint32_t n, uint32_t c, uint32_t t, int& err) {
  std::vector<F> staging((size_t)n * 3);
  std::memcpy(staging.data(), jac_std, staging.size() * sizeof(F));
  std::vector<Affine<F>> table((size_t)t * n);
  std::vector<XYZZ<F>> state(n);
  window_table_enqueue<F>(staging.data(), n, t, (int)c, table.data(), state.data(), &err, nullptr);
  return table;
}

template <class F>
int batch(const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t k, uint32_t stride, uint32_t c, uint32_t t,
          uint32_t S, uint32_t scan_chunk, uint32_t max_rows, uint32_t* out_std) {
  const uint32_t nwin = (255 + c - 1) / c;
  if (t == 0 || t > nwin) return 98;
  int err = 0;
  auto table = make_table<F>(jac_std, n, c, t, err);
  if (err) return 90 + err;
  std::vector<Fr> scalars((size_t)(k - 1) * stride + n);
  std::memcpy(scalars.data(), scalars_std, scalars.size() * sizeof(Fr));
  BatchRun<F> run;
  int rc = msm_batch<F>(table, scalars.data(), n, k, stride, c, t, S, scan_chunk, false, run, max_rows);
  if (rc) return rc;
  for (uint32_t v = 0; v < k; v++) {
    F out[3];
    run_cta(0, 32, 1, [&] { k_finalize<F>(&run.records[v], out); });
    std::memcpy(out_std + (size_t)v * 3 * (sizeof(F) / 4), out, sizeof out);
  }
  return 0;
}

template <class T>
bool same_bytes(const std::vector<T>& a, const std::vector<T>& b) {
  return a.size() == b.size() && std::memcmp(a.data(), b.data(), a.size() * sizeof(T)) == 0;
}

// k = 1 through the batch sequence (vecs = 1; one scan block, or the multi-block scan with scan_chunk) against the
// one-MSM sequence: offsets, slice tables, sorted entries, buckets and the XYZZ record compared byte for byte.
template <class F>
int single_identical(const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t t, uint32_t S,
                     uint32_t scan_chunk) {
  int err = 0;
  auto table = make_table<F>(jac_std, n, c, t, err);
  if (err) return 90 + err;
  std::vector<Fr> scalars(n);
  std::memcpy(scalars.data(), scalars_std, (size_t)n * sizeof(Fr));
  BatchRun<F> one, bat;
  int rc = msm_batch<F>(table, scalars.data(), n, 1, n, c, t, S, 0, true, one);
  if (rc) return rc;
  if ((rc = msm_batch<F>(table, scalars.data(), n, 1, 0, c, t, S, scan_chunk, false, bat))) return rc;
  if (!same_bytes(one.offsets, bat.offsets)) return 1;
  if (!same_bytes(one.slice_off, bat.slice_off)) return 2;
  if (!same_bytes(one.slice_start, bat.slice_start) || !same_bytes(one.slice_end, bat.slice_end)) return 3;
  if (!same_bytes(one.entries, bat.entries)) return 4;
  if (!same_bytes(one.buckets, bat.buckets)) return 5;
  if (c >= 7 && !same_bytes(one.records, bat.records)) return 6;   // same launches: the same record
  F a[3], b[3];
  run_cta(0, 32, 1, [&] { k_finalize<F>(&one.records[0], a); });
  run_cta(0, 32, 1, [&] { k_finalize<F>(&bat.records[0], b); });
  return std::memcmp(a, b, sizeof a) ? 7 : 0;
}
}  // namespace

extern "C" {
// records p < k of sum_i scalars[p*stride + i] * P_i (standard-form Jacobian (x, y, 1), infinity all zero); max_rows: the
// (vector, group) rows per tail launch
int t_msm_batch(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t k, uint32_t stride, uint32_t c,
                uint32_t t, uint32_t S, uint32_t scan_chunk, uint32_t max_rows, uint32_t* out_std) {
  return group == 1 ? batch<Fq>(jac_std, scalars_std, n, k, stride, c, t, S, scan_chunk, max_rows, out_std)
                    : batch<Fq2>(jac_std, scalars_std, n, k, stride, c, t, S, scan_chunk, max_rows, out_std);
}
int t_batch_single_identical(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t t,
                             uint32_t S, uint32_t scan_chunk) {
  return group == 1 ? single_identical<Fq>(jac_std, scalars_std, n, c, t, S, scan_chunk)
                    : single_identical<Fq2>(jac_std, scalars_std, n, c, t, S, scan_chunk);
}
}
