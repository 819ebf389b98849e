// Host-side orchestration of the MSM: window shape, accumulation mode, sort and bucket scratch, and the launch sequence
// of the digit sort, the bucket accumulation and the bucket-sum tails, for one MSM or a batch of scalar vectors over one
// base set.  Every launch goes through B200_LAUNCH / B200_LAUNCH_CTA (poly_host.cuh), so that the SAME host code also
// runs in the CPU test vehicles (tests/host).  Functions return cudaError_t (PCU); the argument checks, with the
// messages b200_last_error reports, are the caller's (capi.cu).
#pragma once
#include <algorithm>
#include <initializer_list>
#include <memory>

#include "bucket_affine.cuh"
#include "poly_host.cuh"

namespace b200 {

constexpr uint32_t kMaxGridY = 65535;    // gridDim.y limit: rows per launch of the (vector, group) tail kernels
constexpr uint32_t kScanTile = 1024;     // threads of a counter-scan block
constexpr uint32_t kScanBlocks = 1024;   // upper bound on the blocks of a batch's counter scan
constexpr int kLPB = 8;

// What the engine takes from its caller: where launches are counted, the B200_CFG_TMA_STAGING mode, an optional
// profiling hook around the accumulation kernels, and launch limits.  The limits default to the library's; the CPU test
// vehicles lower them so that small inputs reach chunked tails, multi-block scans and two-level tree sums.
struct MsmEnv {
  unsigned long long* launch_counter = nullptr;
  int tma_staging = 0;   // 1: staged backward pass in every batched-affine round, 2: only in rounds >= 2
  // called on the accumulation's stream right before it (with the base set's group and the term count) and right after
  void (*prof_begin)(int group, size_t terms, cudaStream_t st) = nullptr;
  void (*prof_end)(cudaStream_t st) = nullptr;
  uint32_t tail_rows = kMaxGridY;         // (vector, group) rows per tail launch
  uint32_t scan_chunk = 64 * kScanTile;   // a batch scans more counters than this with blocks of this many (or more)
  uint32_t tree_sum_max = 1024;           // launch_tree_sum: one block up to this many records,
  uint32_t tree_sum_leaf = 512;           // else this many per first-level block
  void note(unsigned n) const { if (launch_counter) *launch_counter += n; }
};

inline int pick_window_bits(size_t n) {
  // cost model: nwin*n bucket adds (~10 M) + 2*2^(c-1) reduction adds (~14 M), see DESIGN.md §3
  int best = 8;
  double best_cost = 1e300;
  for (int c = 8; c <= 18; c++) {
    double nwin = (255 + c - 1) / c;
    double cost = nwin * (double)n * 10.0 + 2.0 * (double)(1u << (c - 1)) * 14.0 * 4.0;
    if (cost < best_cost) { best_cost = cost; best = c; }
  }
  return best;
}

// The window shape of a base set of n points with c-bit windows, t = B200_CFG_TABLE_WINDOWS as it was at the set's load.
inline MsmShape msm_shape(size_t n, int c, int t) {
  MsmShape sh{};
  sh.n = (uint32_t)n;
  sh.c = (uint32_t)c;
  sh.nwin = (255 + c - 1) / c;
  sh.nbuckets = 1u << (c - 1);
  sh.table_stride = (uint32_t)n;
  // B200_CFG_TABLE_WINDOWS: keep t of the nwin window rows; window w reads row w mod t and feeds bucket group w / t
  sh.rows = t > 0 && (uint32_t)t < sh.nwin ? (uint32_t)t : sh.nwin;
  sh.groups = (sh.nwin + sh.rows - 1) / sh.rows;
  return sh;
}

// Records of launch_bucket_tail's scratch: H rows, K columns and c planes per window group of every scalar vector.
inline size_t bucket_tail_records(const MsmShape& sh) {
  const uint32_t bits = sh.c - 1, kl = (bits + 1) / 2, kh = bits - kl;
  return (size_t)sh.vecs * sh.groups * ((1u << kh) + (1u << kl) + bits + 1);
}

// Output of the digit-recode / counting-sort front end for one scalar vector.  It depends only on the
// scalars and the window shape, so base sets that consume the SAME scalars (A, B1, B2 of a Groth16
// proof) share one SortScratch read-only.
struct SortScratch {
  MsmShape sh{};            // shape it was allocated for (n = capacity)
  DevBuf counts, offsets, cursor, entries, slice_off, slice_start, slice_end;
  uint32_t max_slices = 0;
  uint32_t slice_S = 0;     // > 0: fixed-size slices of S slots (batched-affine mode)
  SliceTables tables() const { return SliceTables{slice_off.as<uint32_t>(), slice_start.as<uint32_t>(), slice_end.as<uint32_t>()}; }
};

// Scratch of the bucket phase: slice sums, buckets, tail records and, for batched-affine accumulation (affine_S > 0),
// ping-pong node buffers, prefix products and per-thread / per-block products.
struct BucketScratch {
  DevBuf slice_out, buckets, partials;
  DevBuf nodeA, nodeB, aff_pre, aff_others, aff_btot, aff_ids;
};

// Front-end and bucket scratch of b200_msm_device_batch on one base set, sized for `vecs` scalar vectors of the set's
// full size.  Allocated on the set's first batch and grown (never shrunk) when a later batch has more vectors.
struct MsmBatch {
  uint32_t vecs = 0;
  SortScratch sort;
  BucketScratch bk;
  DevBuf scan_totals;   // per-block totals of the multi-block counter scan
  cudaEvent_t done = nullptr;   // recorded behind the last batch on the set: a regrowth waits for it, not for the device
  MsmBatch() = default;
  MsmBatch(const MsmBatch&) = delete;
  MsmBatch& operator=(const MsmBatch&) = delete;
  ~MsmBatch() { if (done) cudaEventDestroy(done); }
};

struct Bases {
  int group = 0;  // 1: G1 (Fq), 2: G2 (Fq2)
  size_t n = 0;
  MsmShape sh{};
  DevBuf table;    // [nwin][n] Affine<F>
  // per-base-set scratch of the bucket phase (different base sets may run concurrently)
  DevBuf scalars;  // n * 32 B (host-scalar entry points)
  BucketScratch bk;
  DevBuf result, out_std;
  SortScratch sort;  // own front-end scratch (stand-alone MSMs)
  uint32_t nseg = 0, seg = 0;
  uint32_t affine_S = 0;   // > 0: batched-affine accumulation with slices of affine_S entries
  std::unique_ptr<MsmBatch> batch;   // b200_msm_device_batch scratch (null until the first batch)
  // error word of b200_msm_device on this set: written by the kernels, never read (the call cannot wait for it, and a
  // later call on any object must not report it; see b200snark.h).  Host-pointer MSMs use g_d_err.
  DevBuf d_err;
};

// Device memory held by the buffers (b200_bases_device_bytes / b200_pk_device_bytes).
inline size_t dev_bytes(std::initializer_list<const DevBuf*> bufs) {
  size_t s = 0;
  for (const DevBuf* d : bufs) s += d->p ? d->bytes : 0;
  return s;
}
inline size_t scratch_device_bytes(const SortScratch& ss, const BucketScratch& bk) {
  return dev_bytes({&ss.counts, &ss.offsets, &ss.cursor, &ss.entries, &ss.slice_off, &ss.slice_start, &ss.slice_end,
                    &bk.slice_out, &bk.buckets, &bk.partials, &bk.nodeA, &bk.nodeB, &bk.aff_pre, &bk.aff_others,
                    &bk.aff_btot, &bk.aff_ids});
}
inline size_t bases_device_bytes(const Bases& b) {
  size_t s = dev_bytes({&b.table, &b.scalars, &b.result, &b.out_std, &b.d_err}) + scratch_device_bytes(b.sort, b.bk);
  if (b.batch) s += scratch_device_bytes(b.batch->sort, b.batch->bk) + dev_bytes({&b.batch->scan_totals});
  return s;
}

// slices: every bucket owns >= 1; a bucket above cap = 2*mean entries is cut => at most B + B/2 + 1
inline uint32_t sort_max_slices(const MsmShape& sh, uint32_t slice_S) {
  const size_t entries = (size_t)sh.vecs * sh.nwin * sh.n;
  const uint32_t B = total_buckets(sh);
  return slice_S ? B + (uint32_t)((entries + slice_S - 1) / slice_S) + 2 : B + B / 2 + 2;
}

inline cudaError_t sort_alloc(SortScratch& ss, const MsmShape& sh, uint32_t slice_S) {
  ss.sh = sh;
  ss.slice_S = slice_S;
  size_t entries = (size_t)sh.vecs * sh.nwin * sh.n;
  const uint32_t B = total_buckets(sh);
  PCU(ss.counts.alloc((B + 2) * sizeof(uint32_t)));
  PCU(ss.offsets.alloc((B + 3) * sizeof(uint32_t)));
  PCU(ss.cursor.alloc((B + 2) * sizeof(uint32_t)));
  PCU(ss.entries.alloc(entries * sizeof(uint32_t)));
  ss.max_slices = sort_max_slices(sh, slice_S);
  PCU(ss.slice_off.alloc((B + 3) * sizeof(uint32_t)));
  PCU(ss.slice_start.alloc((size_t)ss.max_slices * sizeof(uint32_t)));
  PCU(ss.slice_end.alloc((size_t)ss.max_slices * sizeof(uint32_t)));
  return cudaSuccess;
}

// Bucket scratch for the shape `sh` (its vecs included) over a sort scratch of max_slices slices: affine_S > 0 adds the
// batched-affine buffers; nseg: segments per window group of the c < 7 tail.
template <class F>
cudaError_t bucket_alloc(BucketScratch& bk, const MsmShape& sh, uint32_t max_slices, uint32_t affine_S, uint32_t nseg) {
  PCU(bk.buckets.alloc((size_t)total_buckets(sh) * sizeof(XYZZ<F>)));
  if (const uint32_t S = affine_S) {
    size_t nsl = max_slices;
    PCU(bk.nodeA.alloc(nsl * (S / 2) * sizeof(Affine<F>)));
    PCU(bk.nodeB.alloc(nsl * (S / 4 ? S / 4 : 1) * sizeof(Affine<F>)));
    PCU(bk.aff_pre.alloc(nsl * (S / 2) * sizeof(F)));
    PCU(bk.aff_ids.alloc(nsl * (S / 2) * sizeof(uint2)));
    size_t nblk_max = (nsl * (S / 2) + kAffBlock * kAffPairs - 1) / (kAffBlock * kAffPairs);
    PCU(bk.aff_others.alloc(nblk_max * kAffBlock * sizeof(F)));
    PCU(bk.aff_btot.alloc(nblk_max * sizeof(F)));
  }
  PCU(bk.slice_out.alloc((size_t)(affine_S ? 1 : max_slices) * sizeof(XYZZ<F>)));
  PCU(bk.partials.alloc(std::max((size_t)sh.vecs * sh.groups * nseg + 1024, bucket_tail_records(sh)) * sizeof(XYZZ<F>)));
  return cudaSuccess;
}

// Accumulation mode of a base set of shape sh: batched affine (6.5 multiplies per add, 3 launches per round) where the
// buckets are populated enough to amortise the rounds, else XYZZ mixed adds (10 multiplies, one launch).  Returns the
// slice size S of the batched-affine mode, 0 for XYZZ.  acc_mode (B200_CFG_ACC_MODE) 1 / 2 forces either.  Auto mode
// keeps a reduced table on XYZZ: the batched-affine node scratch alone is about the size of a full table.  A
// proving-key shard that leaves a rank only a small MSM passes prefer_affine = false (prove_host.cuh).
inline uint32_t affine_slice_size(const MsmShape& sh, int acc_mode, bool prefer_affine) {
  const bool reduced = sh.rows < sh.nwin;
  const bool xyzz_mode = acc_mode == 2 || (acc_mode == 0 && (!prefer_affine || reduced));
  uint32_t S = 0;
  uint64_t mean = ((uint64_t)sh.nwin * sh.n) / total_buckets(sh);
  const uint64_t min_mean = acc_mode == 1 ? 16 : 96;
  if (!xyzz_mode && mean >= min_mean) {
    S = 8;
    while (S < 128 && (uint64_t)S * 2 * 6 <= mean) S *= 2;   // largest power of two <= mean/6, in [8, 128]
  }
  return S;
}

// The set's own sort and bucket scratch (stand-alone MSMs) for its shape and b.affine_S, and the segments of its c < 7
// tail.
template <class F>
cudaError_t bases_scratch(Bases& b) {
  PCU(sort_alloc(b.sort, b.sh, b.affine_S));
  // short latency chain: 4-bucket segments (8 adds + one small scalar mul per thread), then a two-level tree sum
  // (c < 7); nseg segments per window group.  c >= 7: the scratch of launch_bucket_tail.
  b.seg = b.sh.nbuckets >= 256 ? 4 : 1;
  b.nseg = (b.sh.nbuckets + b.seg - 1) / b.seg;
  return bucket_alloc<F>(b.bk, b.sh, b.sort.max_slices, b.affine_S, b.nseg);
}

// Accumulate launch: LPB lanes per bucket slice (2 / 4 / 8 by mean bucket population).  Register budget:
// G1 runs at 128 regs (4 CTAs/SM); occupancy / prefetch variants were no faster — the kernel is bound by the
// IMAD.WIDE issue rate, not by latency hiding.
template <class F, int LPB>
void launch_accumulate_l(const Affine<F>* table, const uint32_t* entries, SliceTables stb, uint32_t m,
                         XYZZ<F>* out, uint32_t max_slices, cudaStream_t st) {
  unsigned grid = nblk((size_t)max_slices * LPB, 128);
  if constexpr (sizeof(F) == sizeof(Fq)) {
    B200_LAUNCH_CTA(B200_K(k_accumulate<F, LPB, 4>), grid, 128, st, table, entries, stb, m, out);
  } else {
    B200_LAUNCH_CTA(B200_K(k_accumulate<F, LPB, 1>), grid, 128, st, table, entries, stb, m, out);
  }
}
template <class F>
void launch_accumulate(int lpb, const Affine<F>* table, const uint32_t* entries, SliceTables stb, uint32_t m,
                       XYZZ<F>* out, uint32_t max_slices, cudaStream_t st) {
  switch (lpb) {
    case 2: launch_accumulate_l<F, 2>(table, entries, stb, m, out, max_slices, st); break;
    case 4: launch_accumulate_l<F, 4>(table, entries, stb, m, out, max_slices, st); break;
    default: launch_accumulate_l<F, 8>(table, entries, stb, m, out, max_slices, st); break;
  }
}

// d_out[0] = sum of partials[0..n): one block if small, else tree_sum_leaf inputs per first-level block + a final block.
// `partials` must have room for n + ceil(n / tree_sum_leaf) records.
template <class F>
void launch_tree_sum(const MsmEnv& env, XYZZ<F>* partials, uint32_t n, XYZZ<F>* d_out, cudaStream_t st) {
  if (n <= env.tree_sum_max) {
    B200_LAUNCH_CTA(k_sum_points<F>, 1, 256, st, partials, n, n, d_out);
    env.note(1);
    return;
  }
  const uint32_t per = env.tree_sum_leaf, nb = (n + per - 1) / per;
  B200_LAUNCH_CTA(k_sum_points<F>, nb, 256, st, partials, n, per, partials + n);
  B200_LAUNCH_CTA(k_sum_points<F>, 1, 256, st, partials + n, nb, nb, d_out);
  env.note(2);
}

// sum_g 2^(c*t*g) sum_b b * S_(g,b) over the bucket array -> one XYZZ record per scalar vector (msm.cuh: rows / columns
// and bit planes of every window group, one Horner chain over the groups of each vector).  `scratch` holds
// bucket_tail_records(sh) records.  Tiny bucket sets keep the segment kernel.
template <class F>
void launch_bucket_tail(const MsmEnv& env, const XYZZ<F>* buckets, const MsmShape& sh, XYZZ<F>* scratch, XYZZ<F>* d_out,
                        cudaStream_t st) {
  const uint32_t bits = sh.c - 1, kl = (bits + 1) / 2, kh = bits - kl, K = 1u << kl, H = 1u << kh, G = sh.groups;
  const uint32_t GV = sh.vecs * G;
  XYZZ<F>* R = scratch;
  XYZZ<F>* C = scratch + (size_t)GV * H;
  XYZZ<F>* planes = C + (size_t)GV * K;
  for_each_tail_chunk(sh, env.tail_rows, [&](uint32_t y0, uint32_t ny) {
    B200_LAUNCH_CTA(k_tail_rowcol<F>, dim3(nblk((size_t)(H + K) * 32, 128), ny), 128, st, buckets + (size_t)y0 * H * K, kl, H,
                    R + (size_t)y0 * H, C + (size_t)y0 * K);
    B200_LAUNCH_CTA(k_tail_planes<F>, dim3(nblk((size_t)(bits + 1) * 32, 128), ny), 128, st, R + (size_t)y0 * H,
                    C + (size_t)y0 * K, kl, kh, planes + (size_t)y0 * (bits + 1));
    env.note(2);
  });
  B200_LAUNCH_CTA(k_tail_horner<F>, sh.vecs, 32, st, planes, bits, d_out, G, sh.c * sh.rows);
  env.note(1);
}

// The c < 7 tail: segment sums (nseg segments of seg buckets) of every window group, each scaled by 2^(c*t*g), then one
// tree sum over all of them (one block per scalar vector in a batch).
template <class F>
void launch_segment_tail(const MsmEnv& env, const MsmShape& sh, uint32_t seg, uint32_t nseg, const XYZZ<F>* buckets,
                         XYZZ<F>* partials, XYZZ<F>* d_out, cudaStream_t st) {
  if (sh.vecs == 1) {
    B200_LAUNCH_CTA(k_bucket_reduce<F>, dim3(nblk(nseg, 128), sh.groups), 128, st, buckets, sh.nbuckets, seg, partials, nseg,
                    sh.c * sh.rows);
    launch_tree_sum<F>(env, partials, sh.groups * nseg, d_out, st);
    return;
  }
  for_each_tail_chunk(sh, env.tail_rows, [&](uint32_t y0, uint32_t ny) {
    B200_LAUNCH_CTA(B200_K(k_bucket_reduce<F, true>), dim3(nblk(nseg, 128), ny), 128, st, buckets + (size_t)y0 * sh.nbuckets,
                    sh.nbuckets, seg, partials + (size_t)y0 * nseg, nseg, sh.c * sh.rows, sh.groups);
    if (y0) env.note(1);   // the caller counts the first k_bucket_reduce
  });
  const uint32_t per = sh.groups * nseg;
  B200_LAUNCH_CTA(k_sum_points<F>, sh.vecs, 256, st, partials, sh.vecs * per, per, d_out);
  env.note(1);
}

// Front end: signed-digit recode + counting sort of n scalars (of each of shape.vecs vectors) into bucket order, in a
// sort scratch allocated for that shape (n <= its capacity).  A standard-form scalar >= r is read as 0 and sets bit 1 of
// *err.  With `scan_totals` (room for kScanBlocks values) a large batch scans its counters with several blocks (one
// more launch).
inline cudaError_t msm_sort(const MsmEnv& env, SortScratch& ss, const MsmShape& shape, const Fr* d_scalars, size_t n,
                            int mont, int* err, cudaStream_t st, unsigned long long* scan_totals = nullptr) {
  MsmShape sh = shape;
  sh.n = (uint32_t)n;
  const uint32_t B = total_buckets(sh);
  uint32_t m = B + 1;  // counts[0] unused (digit 0), buckets 1..B of all window groups
  // slice cap: twice the mean bucket population (uniform scalars never split), at least 4 per lane.  The mean over a
  // batch's buckets is that of one vector.
  uint64_t mean = ((uint64_t)sh.vecs * sh.nwin * n + B - 1) / B;
  uint32_t cap = (uint32_t)(2 * mean < 4 * kLPB ? 4 * kLPB : 2 * mean);
  int fixed = 0;
  if (ss.slice_S) {
    cap = ss.slice_S;
    fixed = 1;
  }
  uint32_t* counts = ss.counts.as<uint32_t>();
  const size_t nterm = (size_t)sh.vecs * n;
  PCU(cudaMemsetAsync(counts, 0, (m + 1) * sizeof(uint32_t), st));
  if (n) B200_LAUNCH(k_digits_count, nblk(nterm, 256), 256, st, d_scalars, sh, mont, counts, err);
  // one block walks up to 64 tiles of counters; beyond that, blocks of 64 tiles each (at most kScanBlocks)
  if (scan_totals && m > env.scan_chunk) {
    uint32_t chunk = env.scan_chunk;
    while ((m + chunk - 1) / chunk > kScanBlocks) chunk *= 2;
    const uint32_t nb = (m + chunk - 1) / chunk;
    B200_LAUNCH_CTA(k_scan_totals, nb, kScanTile, st, counts, m, cap, chunk, scan_totals);
    B200_LAUNCH_CTA(k_scan, nb, kScanTile, st, counts, m, cap, fixed, ss.offsets.as<uint32_t>(), ss.cursor.as<uint32_t>(),
                    ss.tables(), chunk, scan_totals);
    env.note(1);
  } else {
    B200_LAUNCH_CTA(k_scan, 1, kScanTile, st, counts, m, cap, fixed, ss.offsets.as<uint32_t>(), ss.cursor.as<uint32_t>(),
                    ss.tables());
  }
  B200_LAUNCH(k_fill_slices, nblk(m, 256), 256, st, counts, ss.offsets.as<uint32_t>(), m, cap, fixed, ss.tables());
  if (n) B200_LAUNCH(k_digits_scatter, nblk(nterm, 256), 256, st, d_scalars, sh, mont, ss.cursor.as<uint32_t>(),
                     ss.entries.as<uint32_t>(), err);
  env.note(n ? 4 : 2);
  return cudaGetLastError();
}

// Back end: bucket accumulation over the sorted entries of `ss` (sorted with the set's slice size), slice merge,
// weighted bucket reduction and final tree sum -> one XYZZ record in d_out per scalar vector (vecs of them), in the
// scratch `bk`.
template <class F>
cudaError_t bucket_phase(const MsmEnv& env, const Bases* b, const SortScratch& ss, BucketScratch& bk, uint32_t vecs,
                         size_t n_terms, XYZZ<F>* d_out, cudaStream_t st) {
  MsmShape sh = b->sh;
  sh.vecs = vecs;
  const uint32_t B = total_buckets(sh);
  uint32_t m = B + 1;
  XYZZ<F>* buckets = bk.buckets.as<XYZZ<F>>();
  XYZZ<F>* partials = bk.partials.as<XYZZ<F>>();
  SliceTables stb = ss.tables();
  // The out-of-line F_q multiply wins here: the fully inlined madd body (~38 KB of SASS) thrashes the
  // instruction caches.
  if (env.prof_begin) env.prof_begin(b->group, (size_t)vecs * n_terms, st);
  if (b->affine_S) {
    const uint32_t S = b->affine_S;
    uint32_t R = 0;
    while ((1u << R) < S) R++;
    // host-side bound on the live slice count for this call (the exact count lives on the device)
    uint64_t total = (uint64_t)vecs * sh.nwin * n_terms;
    uint64_t nsl_bound = (uint64_t)B + (total + S - 1) / S + 2;
    if (nsl_bound > ss.max_slices) nsl_bound = ss.max_slices;
    AffineRound<F> ar{};
    ar.table = b->table.as<Affine<F>>();
    ar.entries = ss.entries.as<uint32_t>();
    ar.slice_start = stb.slice_start;
    ar.slice_end = stb.slice_end;
    ar.nslices_ptr = stb.slice_off + m;
    ar.pre = bk.aff_pre.as<F>();
    ar.others = bk.aff_others.as<F>();
    ar.btot = bk.aff_btot.as<F>();
    ar.pair_ids = env.tma_staging == 1 ? bk.aff_ids.as<uint2>() : nullptr;
    // node buffers, x- and y-coordinates in separate halves (bucket_affine.cuh NodeBuf)
    const size_t capA = (size_t)ss.max_slices * (S / 2), capB = (size_t)ss.max_slices * (S / 4 ? S / 4 : 1);
    NodeBuf<F> bufs[2] = {{bk.nodeA.as<F>(), bk.nodeA.as<F>() + capA}, {bk.nodeB.as<F>(), bk.nodeB.as<F>() + capB}};
    NodeBuf<F> prev{nullptr, nullptr};
    // all R rounds affine: inside a proof the per-round inversion latency is hidden by the other MSMs' streams
    for (uint32_t r = 1; r <= R; r++) {
      ar.round = r;
      ar.q_log = R - r;
      ar.prev = prev;
      ar.out = bufs[(r - 1) & 1];
      uint64_t npairs_max = nsl_bound << ar.q_log;
      unsigned nb = (unsigned)((npairs_max + kAffBlock * kAffPairs - 1) / (kAffBlock * kAffPairs));
      const bool staged = env.tma_staging == 1 || (env.tma_staging == 2 && r >= 2);
      // CTAs/SM bounds = register caps (forward 8 + backward 5 CTAs/SM for G1, 4 + 4 for G2); chosen by a sweep on an
      // earlier target and not re-swept on the H100
      if (sizeof(F) == 32) {
        B200_LAUNCH_CTA(B200_K(k_affine_forward<F, kAffPairs, 8>), nb, kAffBlock, st, ar);
        B200_LAUNCH_CTA(k_affine_invert<F>, nblk((size_t)nb * 32, 128), 128, st, ar.btot, nb);
        if (staged) B200_LAUNCH_CTA_SMEM(B200_K(k_affine_backward_staged<F, kAffPairs, 5>), nb, kAffBlock, AffStageLayout<F>::kSmem, st, ar);
        else B200_LAUNCH(B200_K(k_affine_backward<F, kAffPairs, 5>), nb, kAffBlock, st, ar);
      } else {
        B200_LAUNCH_CTA(B200_K(k_affine_forward<F, kAffPairs, 4>), nb, kAffBlock, st, ar);
        B200_LAUNCH_CTA(k_affine_invert<F>, nblk((size_t)nb * 32, 128), 128, st, ar.btot, nb);
        if (staged) B200_LAUNCH_CTA_SMEM(B200_K(k_affine_backward_staged<F, kAffPairs, 4>), nb, kAffBlock, AffStageLayout<F>::kSmem, st, ar);
        else B200_LAUNCH(B200_K(k_affine_backward<F, kAffPairs, 4>), nb, kAffBlock, st, ar);
      }
      prev = ar.out;
      env.note(3);
    }
    if (env.prof_end) env.prof_end(st);
    B200_LAUNCH_CTA(k_merge_slices_affine<F>, nblk(B, 128), 128, st, prev, stb, B, buckets);
    if (sh.c >= 7) {
      launch_bucket_tail<F>(env, buckets, sh, partials, d_out, st);
      env.note(1);
    } else {
      launch_segment_tail<F>(env, sh, b->seg, b->nseg, buckets, partials, d_out, st);
      env.note(2);
    }
    return cudaGetLastError();
  }
  uint64_t mean = ((uint64_t)vecs * sh.nwin * n_terms + B - 1) / B;   // that of one vector
  int lpb = mean >= 384 ? 8 : (mean >= 96 ? 4 : 2);
  launch_accumulate<F>(lpb, b->table.as<Affine<F>>(), ss.entries.as<uint32_t>(), stb, m,
                       bk.slice_out.as<XYZZ<F>>(), ss.max_slices, st);
  if (env.prof_end) env.prof_end(st);
  B200_LAUNCH_CTA(k_merge_slices<F>, nblk(B, 128), 128, st, bk.slice_out.as<XYZZ<F>>(), stb, B, buckets);
  if (sh.c >= 7) {
    launch_bucket_tail<F>(env, buckets, sh, partials, d_out, st);
    env.note(1);
  } else {
    launch_segment_tail<F>(env, sh, b->seg, b->nseg, buckets, partials, d_out, st);
    env.note(3);
  }
  return cudaGetLastError();
}

// One MSM's back end in the set's own bucket scratch (4 launches + the tail), over a sort of the set's shape and slices.
template <class F>
cudaError_t msm_buckets(const MsmEnv& env, Bases* b, const SortScratch& ss, size_t n_terms, XYZZ<F>* d_out, cudaStream_t st) {
  return bucket_phase<F>(env, b, ss, b->bk, 1, n_terms, d_out, st);
}

// One MSM of n <= b->n terms in the set's own scratch.
template <class F>
cudaError_t msm_enqueue(const MsmEnv& env, Bases* b, const Fr* d_scalars, size_t n, int mont, XYZZ<F>* d_out, int* err,
                        cudaStream_t st) {
  PCU(msm_sort(env, b->sort, b->sh, d_scalars, n, mont, err, st));
  return msm_buckets<F>(env, b, b->sort, n, d_out, st);
}

// ---- batches: k scalar vectors over one base set -----------------------------------------------------------------
// Term i of vector p is scalar p*stride + i times base i; vector p's digits go to its own window groups, so one recode,
// one counting sort, one accumulation and one tail serve all k vectors.  Populations per bucket, and so the slice cap,
// the lanes per bucket and the accumulation kernel, are those of one vector.
inline bool batch_fits(const MsmShape& sh, size_t k, size_t n) {
  return (uint64_t)k * sh.nwin * n < (1ull << 31) && (uint64_t)k * total_buckets(sh) + 3 < (1ull << 31);
}
inline bool batch_fits(const Bases* b, size_t k, size_t n) { return batch_fits(b->sh, k, n); }

// The batch scratch of `b` for k vectors of n terms: allocated on the first batch, regrown to the larger of the old and
// the new capacity in each dimension when a batch exceeds it.  Before the old buffers are freed the host waits for the
// set's last batch (its `done` event); batches on one set are ordered on one stream (b200snark.h), so nothing else of
// this set can still read them, and work on other sets and prove contexts is not waited for.
// with_sort = false (a proving-key set whose batches reuse another set's sort of the same scalars): bucket scratch
// only, for that sort's slices; the shape is recorded in `sort.sh`, and nothing else of `sort` is allocated.
template <class F>
cudaError_t batch_scratch(Bases* b, uint32_t k, uint32_t n, bool with_sort = true) {
  if (n == 0) n = 1;
  if (b->batch && b->batch->vecs >= k && b->batch->sort.sh.n >= n && (!with_sort || b->batch->sort.entries.p)) return cudaSuccess;
  if (b->batch) {
    PCU(cudaEventSynchronize(b->batch->done));
    const uint32_t k2 = std::max(k, b->batch->vecs), n2 = std::max(n, b->batch->sort.sh.n);
    if (batch_fits(b, k2, n2)) k = k2, n = n2;   // else: exactly this batch's size
  }
  b->batch.reset();
  auto mb = std::make_unique<MsmBatch>();
  MsmShape sh = b->sh;
  sh.n = n;
  sh.vecs = k;
  if (with_sort) {
    PCU(sort_alloc(mb->sort, sh, b->affine_S));
    PCU(mb->scan_totals.alloc(kScanBlocks * sizeof(unsigned long long)));
  } else {
    mb->sort.sh = sh;
  }
  PCU(bucket_alloc<F>(mb->bk, sh, sort_max_slices(sh, b->affine_S), b->affine_S, b->nseg));
  PCU(cudaEventCreateWithFlags(&mb->done, cudaEventDisableTiming));
  mb->vecs = k;
  b->batch = std::move(mb);
  return cudaSuccess;
}

// k MSMs of n <= b->n terms (vector p at d_scalars + p*stride) in the set's batch scratch, grown as needed; the caller
// has checked batch_fits(b, k, n).
template <class F>
cudaError_t msm_batch_enqueue(const MsmEnv& env, Bases* b, const Fr* d_scalars, size_t n, size_t k, size_t stride, int mont,
                              XYZZ<F>* d_out, int* err, cudaStream_t st) {
  PCU(batch_scratch<F>(b, (uint32_t)k, (uint32_t)n));
  MsmBatch& mb = *b->batch;
  MsmShape sh = b->sh;
  sh.vecs = (uint32_t)k;
  sh.vec_stride = (uint32_t)stride;
  PCU(msm_sort(env, mb.sort, sh, d_scalars, n, mont, err, st, mb.scan_totals.as<unsigned long long>()));
  PCU(bucket_phase<F>(env, b, mb.sort, mb.bk, (uint32_t)k, n, d_out, st));
  return cudaEventRecord(mb.done, st);
}

}  // namespace b200
