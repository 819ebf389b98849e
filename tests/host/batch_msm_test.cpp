// CPU test vehicle for batches of MSMs over one base set (b200_msm_device_batch; g++, csrc/host_stub): k scalar vectors
// through the library's MSM engine (msm_host.cuh: msm_batch_enqueue — the batched digit recode and counting sort, vector
// p's digits in window groups p*G .. p*G + G - 1, the multi-block counter scan, both accumulation kernels, the slice
// merge, and the per-vector tails: rows / columns and bit planes over (vector, group) as blockIdx.y, one Horner chain per
// vector as blockIdx.x; or, for c < 7, scaled segment sums and one tree-sum block per vector).  k = 1 is also compared
// with the engine's one-MSM path (msm_enqueue) array by array.  Reuses the CTA emulation of host_kernel_test.cpp.
// Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"

namespace {
// k vectors of n scalars (vector p at scalars + p*stride) over a table of t rows; scan_chunk > 0: the counter scan in
// blocks of scan_chunk counters (k_scan_totals + k_scan), else one block; the (vector, group) tail kernels in launches of
// at most max_rows rows (65535 on the device; a small max_rows puts chunk boundaries inside a batch).
template <class F>
int batch(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t k, uint32_t stride, uint32_t c,
          uint32_t t, uint32_t S, uint32_t scan_chunk, uint32_t max_rows, uint32_t* out_std) {
  if (t == 0 || t > (255 + c - 1) / c) return 98;
  int err = 0;
  Bases b;
  int rc = make_bases<F>(b, group, jac_std, n, c, t, S, &err);
  if (err) return 90 + err;
  if (rc) return rc;
  std::vector<Fr> scalars((size_t)(k - 1) * stride + n);
  std::memcpy(scalars.data(), scalars_std, scalars.size() * sizeof(Fr));
  std::vector<XYZZ<F>> records(k);
  const MsmEnv env = test_env(0, max_rows, scan_chunk);
  if (msm_batch_enqueue<F>(env, &b, scalars.data(), n, k, stride, 0, records.data(), &err, nullptr)) return 95;
  if (err) return 100 + err;
  MsmShape sh = b.sh;
  sh.vecs = k;
  if ((rc = check_sort(b.batch->sort, sh))) return rc;
  for (uint32_t v = 0; v < k; v++) finalize_std<F>(records[v], out_std + (size_t)v * 3 * (sizeof(F) / 4));
  return 0;
}

// What a sort and a bucket phase leave behind: offsets, slice tables, sorted entries and buckets (their live parts).
struct SortRun {
  std::vector<uint8_t> offsets, slice_off, slices, entries, buckets;
};
template <class F>
SortRun take_run(const SortScratch& ss, const BucketScratch& bk, const MsmShape& sh) {
  const uint32_t m = total_buckets(sh) + 1, nsl = ss.tables().slice_off[m], ne = ss.offsets.as<uint32_t>()[m];
  auto bytes = [](const DevBuf& d, size_t off, size_t len) {
    const uint8_t* p = d.as<uint8_t>() + off;
    return std::vector<uint8_t>(p, p + len);
  };
  SortRun r;
  r.offsets = bytes(ss.offsets, 0, (m + 1) * sizeof(uint32_t));
  r.slice_off = bytes(ss.slice_off, 0, (m + 1) * sizeof(uint32_t));
  r.slices = bytes(ss.slice_start, 0, nsl * sizeof(uint32_t));
  auto ends = bytes(ss.slice_end, 0, nsl * sizeof(uint32_t));
  r.slices.insert(r.slices.end(), ends.begin(), ends.end());
  r.entries = bytes(ss.entries, 0, ne * sizeof(uint32_t));
  r.buckets = bytes(bk.buckets, 0, (m - 1) * sizeof(XYZZ<F>));
  return r;
}

// k = 1 through the engine's batch path (msm_batch_enqueue: one scan block, or the multi-block scan with scan_chunk)
// against its one-MSM path (msm_enqueue): offsets, slice tables, sorted entries, buckets and the XYZZ record compared
// byte for byte.
template <class F>
int single_identical(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t t,
                     uint32_t S, uint32_t scan_chunk) {
  int err = 0;
  Bases b;
  int rc = make_bases<F>(b, group, jac_std, n, c, t, S, &err);
  if (err) return 90 + err;
  if (rc) return rc;
  std::vector<Fr> scalars(n);
  std::memcpy(scalars.data(), scalars_std, (size_t)n * sizeof(Fr));
  XYZZ<F> one_rec, bat_rec;
  if (msm_enqueue<F>(test_env(0), &b, scalars.data(), n, 0, &one_rec, &err, nullptr)) return 95;
  if ((rc = check_sort(b.sort, b.sh))) return rc;
  const SortRun one = take_run<F>(b.sort, b.bk, b.sh);
  if (msm_batch_enqueue<F>(test_env(0, kMaxGridY, scan_chunk), &b, scalars.data(), n, 1, 0, 0, &bat_rec, &err, nullptr)) return 95;
  if (err) return 100 + err;
  if ((rc = check_sort(b.batch->sort, b.sh))) return rc;
  const SortRun bat = take_run<F>(b.batch->sort, b.batch->bk, b.sh);
  if (one.offsets != bat.offsets) return 1;
  if (one.slice_off != bat.slice_off) return 2;
  if (one.slices != bat.slices) return 3;
  if (one.entries != bat.entries) return 4;
  if (one.buckets != bat.buckets) return 5;
  if (c >= 7 && std::memcmp(&one_rec, &bat_rec, sizeof one_rec)) return 6;   // same launches: the same record
  uint32_t a[3 * sizeof(F) / 4], z[3 * sizeof(F) / 4];
  finalize_std<F>(one_rec, a);
  finalize_std<F>(bat_rec, z);
  return std::memcmp(a, z, sizeof a) ? 7 : 0;
}
}  // namespace

extern "C" {
// records p < k of sum_i scalars[p*stride + i] * P_i (standard-form Jacobian (x, y, 1), infinity all zero); max_rows: the
// (vector, group) rows per tail launch
int t_msm_batch(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t k, uint32_t stride, uint32_t c,
                uint32_t t, uint32_t S, uint32_t scan_chunk, uint32_t max_rows, uint32_t* out_std) {
  return group == 1 ? batch<Fq>(group, jac_std, scalars_std, n, k, stride, c, t, S, scan_chunk, max_rows, out_std)
                    : batch<Fq2>(group, jac_std, scalars_std, n, k, stride, c, t, S, scan_chunk, max_rows, out_std);
}
int t_batch_single_identical(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t t,
                             uint32_t S, uint32_t scan_chunk) {
  return group == 1 ? single_identical<Fq>(group, jac_std, scalars_std, n, c, t, S, scan_chunk)
                    : single_identical<Fq2>(group, jac_std, scalars_std, n, c, t, S, scan_chunk);
}
}
