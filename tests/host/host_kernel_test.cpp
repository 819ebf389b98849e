// CPU test vehicle for the per-thread bucket kernels of bucket_affine.cuh (g++, csrc/host_stub): the backward-pass
// variants — the product kernel and the experiment kernels k_affine_backward_lr / _sp — are run one emulated thread at
// a time over all rounds of a small slice forest, against a plain host restatement of the forward pass.  What this
// checks is the kernels' own index logic (pair <-> slice <-> entry mapping, staging queues, fast/slow path split,
// sign and infinity handling); the field arithmetic underneath is covered by host_arith_test.cpp.  Whole MSMs run the
// library's own MSM engine (msm_host.cuh) on the emulated kernels.
// Test infrastructure only: never linked into libb200snark.
#include "host_stub/cuda_runtime.h"

#include <pthread.h>

#include <thread>
#include <vector>

#include "bucket_affine.cuh"
#include "ntt.cuh"

// the host orchestration (poly_host.cuh, qap_sparse.cuh, msm_host.cuh) launches through these: sequential emulated
// threads for plain kernels, one OS thread per CUDA thread for kernels that synchronise inside a CTA (with `smem` bytes of
// dynamic shared memory per CTA)
template <class K> void stub_launch_threads(dim3 grid, unsigned nthreads, K k);
template <class K> void stub_launch_cta(dim3 grid, unsigned nthreads, size_t smem, K k);
#define B200_LAUNCH(kernel, grid, block, stream, ...) stub_launch_threads(dim3(grid), (unsigned)(block), [&] { kernel(__VA_ARGS__); })
#define B200_LAUNCH_CTA(kernel, grid, block, stream, ...) stub_launch_cta(dim3(grid), (unsigned)(block), 0, [&] { kernel(__VA_ARGS__); })
#define B200_LAUNCH_CTA_SMEM(kernel, grid, block, smem, stream, ...) \
  stub_launch_cta(dim3(grid), (unsigned)(block), (size_t)(smem), [&] { kernel(__VA_ARGS__); })
#include "qap_sparse.cuh"
#include "fixed_base.cuh"
#include "msm_host.cuh"
#include "pairing_warp.cuh"
#include "glv.cuh"

using namespace b200;

// ---- CTA-at-a-time emulation: one OS thread per CUDA thread, barriers for __syncthreads and the warp shuffles ------
namespace {
constexpr int kMaxWarps = 32;
pthread_barrier_t g_block_bar, g_warp_bar[kMaxWarps];
uint32_t g_xchg[kMaxWarps][32];
bool g_cta_mode = false;
}  // namespace
void stub_syncthreads() {
  if (!g_cta_mode) stub_abort("__syncthreads outside run_cta");
  pthread_barrier_wait(&g_block_bar);
}
uint32_t stub_shfl(uint32_t v, int arg, int mode, int width) {
  if (!g_cta_mode) stub_abort("warp shuffle outside run_cta");
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  g_xchg[warp][lane] = v;
  pthread_barrier_wait(&g_warp_bar[warp]);
  int seg = lane & ~(width - 1), pos = lane & (width - 1), src;
  if (mode == 0) src = seg + (arg & (width - 1));
  else if (mode == 1) src = pos - arg >= 0 ? lane - arg : lane;
  else src = pos + arg < width ? lane + arg : lane;
  uint32_t r = g_xchg[warp][src];
  pthread_barrier_wait(&g_warp_bar[warp]);
  return r;
}
void stub_syncwarp() {
  if (g_cta_mode) pthread_barrier_wait(&g_warp_bar[threadIdx.x >> 5]);
}
unsigned stub_ballot(int pred) {
  if (!g_cta_mode) stub_abort("__ballot_sync outside run_cta");
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  g_xchg[warp][lane] = pred ? 1u : 0u;
  pthread_barrier_wait(&g_warp_bar[warp]);
  unsigned r = 0;
  for (int l = 0; l < 32; l++) r |= g_xchg[warp][l] << l;
  pthread_barrier_wait(&g_warp_bar[warp]);
  return r;
}
namespace {
// run `kernel()` for every thread of CTA (b, y) of an nblocks x ny grid (nthreads a multiple of 32, <= 1024), with
// `smem` as its dynamic shared memory
template <class K>
void run_cta(unsigned b, unsigned nthreads, unsigned nblocks, K kernel, unsigned y = 0, unsigned ny = 1, uint8_t* smem = nullptr) {
  pthread_barrier_init(&g_block_bar, nullptr, nthreads);
  for (unsigned w = 0; w < nthreads / 32; w++) pthread_barrier_init(&g_warp_bar[w], nullptr, 32);
  g_cta_mode = true;
  std::vector<std::thread> th;
  for (unsigned t = 0; t < nthreads; t++)
    th.emplace_back([=] {
      threadIdx.x = t;
      blockIdx.x = b;
      blockIdx.y = y;
      blockDim.x = nthreads;
      gridDim.x = nblocks;
      gridDim.y = ny;
      g_stub_dyn_smem = smem;
      kernel();
    });
  for (auto& x : th) x.join();
  g_cta_mode = false;
  pthread_barrier_destroy(&g_block_bar);
  for (unsigned w = 0; w < nthreads / 32; w++) pthread_barrier_destroy(&g_warp_bar[w]);
}

template <class F>
F load_std(const uint32_t* p) {
  F v;
  std::memcpy(&v, p, sizeof(F));
  return v.to_mont();
}
template <class F>
void store_std(uint32_t* p, const F& v) {
  F s = v.from_mont();
  std::memcpy(p, &s, sizeof(F));
}

// forward pass, restated: pre[p], others[thread], btot[block] exactly as k_affine_forward defines them
template <class F, int T>
void forward_reference(const AffineRound<F>& a, uint32_t npairs, unsigned nb) {
  for (unsigned b = 0; b < nb; b++) {
    uint32_t block_base = b * (kAffBlock * T);
    if (block_base >= npairs) {
      a.btot[b] = F::one();
      continue;
    }
    std::vector<F> tot(kAffBlock, F::one());
    for (unsigned t = 0; t < kAffBlock; t++) {
      F run = F::one();
      for (int k = 0; k < T; k++) {
        uint32_t p = block_base + k * kAffBlock + t;
        Affine<F> P, Q;
        F d;
        if (aff_operands(a, p, npairs, P, Q)) {
          aff_denominator(P, Q, d);
          F dx;                                   // the x-only forward path must agree with the full one
          if (!aff_forward_denominator(a, p, npairs, dx) || !(dx == d)) std::abort();
          a.pre[p] = run;
          run = run * d;
        }
      }
      tot[t] = run;
    }
    F all = F::one();
    for (unsigned t = 0; t < kAffBlock; t++) all = all * tot[t];
    for (unsigned t = 0; t < kAffBlock; t++) {
      F o = F::one();
      for (unsigned u = 0; u < kAffBlock; u++)
        if (u != t) o = o * tot[u];
      a.others[b * kAffBlock + t] = o;
    }
    a.btot[b] = all.inverse();                    // k_affine_invert
  }
}

// the forward kernels themselves (block scan included), CTA by CTA: 0 product kernel, 1 L2-prefetch variant, 2 _sp
template <class F, int T>
void run_forward(int variant, const AffineRound<F>& a, unsigned nb) {
  for (unsigned b = 0; b < nb; b++)
    run_cta(b, kAffBlock, nb, [&] {
      (void)variant;
      k_affine_forward<F, T, 1>(a);
    });
  for (unsigned b = 0; b < nb; b++) a.btot[b] = a.btot[b].inverse();   // k_affine_invert
}

template <class F, int T>
void run_backward(int variant, const AffineRound<F>& a, unsigned nb) {
  if (variant == 1) {   // the staged kernel (TMA bulk copies / cp.async gathers emulated as synchronous copies), CTA by CTA
    static std::vector<uint8_t> smem;
    smem.assign(AffStageLayout<F>::kSmem + 128, 0);
    uint8_t* base = smem.data();
    for (unsigned b = 0; b < nb; b++)
      run_cta(b, kAffBlock, nb, [&] {
        g_stub_dyn_smem = base;
        k_affine_backward_staged<F, T, 1>(a);
      });
    return;
  }
  blockDim.x = kAffBlock;
  gridDim.x = nb;
  for (unsigned b = 0; b < nb; b++)
    for (unsigned t = 0; t < kAffBlock; t++) {
      blockIdx.x = b;
      threadIdx.x = t;
      (void)variant;
      k_affine_backward<F, T, 1>(a);
    }
}

template <class F, int T>
int affine_rounds(int variant, int fwd_variant, const uint32_t* table_std, uint32_t n_pts, const uint32_t* entries, const uint32_t* slice_start,
                  const uint32_t* slice_end, uint32_t nslices, uint32_t R, uint32_t* out_std) {
  constexpr int W = sizeof(F) / 4;
  std::vector<Affine<F>> table(n_pts);
  for (uint32_t i = 0; i < n_pts; i++) {
    table[i].x = load_std<F>(table_std + (size_t)i * 2 * W);
    table[i].y = load_std<F>(table_std + (size_t)i * 2 * W + W);
  }
  const uint32_t S = 1u << R;
  const size_t cap = (size_t)nslices * (S / 2);
  std::vector<F> bufA(2 * cap), bufB(2 * cap);        // x-coordinates in the first half, y-coordinates in the second (NodeBuf)
  std::vector<F> pre((size_t)nslices * (S / 2));
  std::vector<uint2> ids((size_t)nslices * (S / 2));
  unsigned nb_max = (nslices * (S / 2) + kAffBlock * T - 1) / (kAffBlock * T);
  std::vector<F> others((size_t)nb_max * kAffBlock), btot(nb_max);
  AffineRound<F> ar{};
  ar.table = table.data();
  ar.entries = entries;
  ar.slice_start = slice_start;
  ar.slice_end = slice_end;
  ar.nslices_ptr = &nslices;
  ar.pre = pre.data();
  ar.others = others.data();
  ar.btot = btot.data();
  ar.pair_ids = ids.data();
  NodeBuf<F> prev{nullptr, nullptr};
  NodeBuf<F> bufs[2] = {{bufA.data(), bufA.data() + cap}, {bufB.data(), bufB.data() + cap}};
  for (uint32_t r = 1; r <= R; r++) {
    ar.round = r;
    ar.q_log = R - r;
    ar.prev = prev;
    ar.out = bufs[(r - 1) & 1];
    uint32_t npairs = nslices << ar.q_log;
    unsigned nb = (npairs + kAffBlock * T - 1) / (kAffBlock * T);
    if (fwd_variant < 0) {
      forward_reference<F, T>(ar, npairs, nb);
    } else {
      // kernel forward pass, checked against the restatement (pre, others, 1/btot) before it is consumed
      run_forward<F, T>(fwd_variant, ar, nb);
      std::vector<F> pre_k(pre), others_k(others), btot_k(btot);
      forward_reference<F, T>(ar, npairs, nb);
      for (uint32_t p = 0; p < npairs; p++)
        if (!(pre_k[p] == pre[p])) return 10 + (int)r;
      for (unsigned b = 0; b < nb; b++) {
        if (!(btot_k[b] == btot[b])) return 20 + (int)r;
        if (b * (kAffBlock * T) >= npairs) continue;
        for (unsigned t = 0; t < kAffBlock; t++)
          if (!(others_k[b * kAffBlock + t] == others[b * kAffBlock + t])) return 30 + (int)r;
      }
    }
    run_backward<F, T>(variant, ar, nb);
    prev = ar.out;
  }
  for (uint32_t s = 0; s < nslices; s++) {
    store_std(out_std + (size_t)s * 2 * W, prev.x[s]);
    store_std(out_std + (size_t)s * 2 * W + W, prev.y[s]);
  }
  return 0;
}

template <class K>
void run_threads(dim3 grid, unsigned nthreads, K kernel) {  // kernels without barriers: one thread at a time
  blockDim.x = nthreads;
  gridDim.x = grid.x;
  gridDim.y = grid.y;
  for (unsigned y = 0; y < grid.y; y++)
    for (unsigned b = 0; b < grid.x; b++)
      for (unsigned t = 0; t < nthreads; t++) {
        blockIdx.x = b;
        blockIdx.y = y;
        threadIdx.x = t;
        kernel();
      }
}
inline unsigned cdiv(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

// The MSM engine's settings in the vehicles: launch limits lowered so that small inputs reach two-level tree sums (above
// 64 records, 32 per first-level block), chunked tails (max_rows rows per launch) and multi-block counter scans (blocks of
// scan_chunk counters; 0: one block); staging = B200_CFG_TMA_STAGING.
inline MsmEnv test_env(int staging, uint32_t max_rows = kMaxGridY, uint32_t scan_chunk = 0) {
  MsmEnv env;
  env.tma_staging = staging;
  env.tail_rows = max_rows;
  env.scan_chunk = scan_chunk ? scan_chunk : 0xffffffffu;
  env.tree_sum_max = 64;
  env.tree_sum_leaf = 32;
  return env;
}

// A base set as bases_create makes one, on the emulated device: n standard-form Jacobian points, c-bit windows, t table
// rows (0: all) built by window_table_enqueue, and the engine's scratch for batched-affine slices of S entries (0: XYZZ).
// Bit 0 of err: a coordinate >= q.
template <class F>
int make_bases(Bases& b, int group, const uint32_t* jac_std, uint32_t n, uint32_t c, uint32_t t, uint32_t S, int* err) {
  b.group = group;
  b.n = n;
  b.sh = msm_shape(n, (int)c, (int)t);
  std::vector<F> staging((size_t)n * 3);
  std::memcpy(staging.data(), jac_std, staging.size() * sizeof(F));
  std::vector<XYZZ<F>> state(n);
  if (b.table.alloc((size_t)b.sh.rows * n * sizeof(Affine<F>))) return 91;
  window_table_enqueue<F>(staging.data(), n, b.sh.rows, (int)c, b.table.as<Affine<F>>(), state.data(), err, nullptr);
  b.affine_S = S;
  return bases_scratch<F>(b) ? 92 : 0;
}

// The sort's own invariants: every entry reads one of the `rows` stored table rows of a base < n, each bucket is filled
// exactly to the next one's offset, and the slices fit the scratch.
inline int check_sort(const SortScratch& ss, const MsmShape& sh) {
  const uint32_t m = total_buckets(sh) + 1;
  const uint32_t *offsets = ss.offsets.as<uint32_t>(), *cursor = ss.cursor.as<uint32_t>(), *entries = ss.entries.as<uint32_t>();
  for (uint32_t e = 0; e < offsets[m]; e++)
    if ((entries[e] >> 1) >= (size_t)sh.rows * sh.table_stride || (entries[e] >> 1) % sh.table_stride >= sh.n) return 96;
  for (uint32_t b = 1; b < m; b++)
    if (cursor[b] != offsets[b + 1]) return 97;
  return ss.tables().slice_off[m] > ss.max_slices ? 99 : 0;
}

template <class F>
void finalize_std(const XYZZ<F>& rec, uint32_t* out_std) {
  F out[3];
  run_cta(0, 32, 1, [&] { k_finalize<F>(&rec, out); });
  std::memcpy(out_std, out, sizeof out);
}

// Back end of an MSM after the accumulation: slices -> buckets (k_merge_slices_affine), then the engine's tails:
// seg = 0 the rows / columns + bit planes + Horner tail (launch_bucket_tail, nbuckets = 2^(c-1)), else segment sums of seg
// buckets and a one- or two-level tree sum (launch_segment_tail); normalisation (k_finalize).
template <class F>
int msm_tail(const uint32_t* slice_pts_std, const uint32_t* slice_off, uint32_t nbuckets, uint32_t seg, uint32_t* out_std) {
  constexpr int W = sizeof(F) / 4;
  uint32_t nsl = slice_off[nbuckets + 1];
  const size_t cap_t = nsl ? nsl : 1;
  std::vector<F> pts(2 * cap_t);
  for (uint32_t i = 0; i < nsl; i++) {
    pts[i] = load_std<F>(slice_pts_std + (size_t)i * 2 * W);
    pts[cap_t + i] = load_std<F>(slice_pts_std + (size_t)i * 2 * W + W);
  }
  std::vector<XYZZ<F>> buckets(nbuckets);
  SliceTables st{const_cast<uint32_t*>(slice_off), nullptr, nullptr};
  unsigned nb = (nbuckets + 127) / 128;
  for (unsigned b = 0; b < nb; b++) run_cta(b, 128, nb, [&] { k_merge_slices_affine<F>(NodeBuf<F>{pts.data(), pts.data() + cap_t}, st, nbuckets, buckets.data()); });
  const MsmEnv env = test_env(0);
  XYZZ<F> total;
  if (seg == 0) {
    uint32_t bits = 0;
    while ((1u << bits) < nbuckets) bits++;
    if ((1u << bits) != nbuckets) return 7;
    const MsmShape sh = msm_shape(0, (int)bits + 1, 0);
    std::vector<XYZZ<F>> scratch(bucket_tail_records(sh));
    launch_bucket_tail<F>(env, buckets.data(), sh, scratch.data(), &total, nullptr);
  } else {
    MsmShape sh{};   // one window group of nbuckets buckets
    sh.nbuckets = nbuckets;
    const uint32_t nseg = (nbuckets + seg - 1) / seg;
    std::vector<XYZZ<F>> partials((size_t)nseg + 1024);
    launch_segment_tail<F>(env, sh, seg, nseg, buckets.data(), partials.data(), &total, nullptr);
  }
  finalize_std<F>(total, out_std);
  return 0;
}

// ---- a whole MSM through the library's engine (msm_host.cuh: msm_enqueue — digit recode, counting sort, slice
// tables, bucket accumulation (batched-affine rounds when S != 0, else the XYZZ kernel with 2, 4 or 8 lanes per slice),
// slice merge, bucket tail) over a base set built as bases_create builds it, then k_finalize.  G1 runs the staged
// backward pass in every round (B200_CFG_TMA_STAGING 1), G2 from round 2 on (2).
template <class F>
int msm_full(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t S, uint32_t* out_std) {
  int err = 0;
  Bases b;
  int rc = make_bases<F>(b, group, jac_std, n, c, 0, S, &err);
  if (rc) return rc;
  std::vector<Fr> scalars(n);
  std::memcpy(scalars.data(), scalars_std, (size_t)n * sizeof(Fr));
  XYZZ<F> rec;
  if (msm_enqueue<F>(test_env(group == 1 ? 1 : 2), &b, scalars.data(), n, 0, &rec, &err, nullptr)) return 95;
  if (err) return 100 + err;
  if ((rc = check_sort(b.sort, b.sh))) return rc;
  finalize_std<F>(rec, out_std);
  return 0;
}
// out = a * b over F_r with the NTT kernels, in the order of PolyCtx::forward / pointwise / inverse_unscaled
// (poly_host.cuh): load + Montgomery, DIF stages, pointwise product scaled by 1/N, DIT stages, store.
int poly_mul_kernels(const uint32_t* a_std, uint32_t la, const uint32_t* b_std, uint32_t lb, uint32_t* out_std) {
  uint32_t lo = la + lb - 1;
  int logn = 1;
  while ((1u << logn) < lo) logn++;
  uint32_t N = 1u << logn, n_half = N >> 1;
  Fr root;
  for (int i = 0; i < 8; i++) root.l[i] = FrParams::ROOT(i);
  Fr w = root;
  for (int i = 0; i < FrParams::TWO_ADICITY - logn; i++) w = w.sqr();
  Fr w_inv = w.inverse();
  Fr nf = Fr::zero();
  nf.l[0] = N;
  Fr n_inv = nf.to_mont().inverse();
  std::vector<Fr> tw(n_half), tw_inv(n_half), A(N), B(N), src_a(la), src_b(lb), out(lo);
  std::memcpy(src_a.data(), a_std, (size_t)la * sizeof(Fr));
  std::memcpy(src_b.data(), b_std, (size_t)lb * sizeof(Fr));
  int err = 0;
  run_threads(cdiv(n_half, 256), 256, [&] { k_twiddles(tw.data(), n_half, w); });
  run_threads(cdiv(n_half, 256), 256, [&] { k_twiddles(tw_inv.data(), n_half, w_inv); });
  run_threads(cdiv(N, 256), 256, [&] { k_poly_load(src_a.data(), la, la, 0, 0, A.data(), N, &err); });
  run_threads(cdiv(N, 256), 256, [&] { k_poly_load(src_b.data(), lb, lb, 0, 0, B.data(), N, &err); });
  for (Fr* d : {A.data(), B.data()})
    for (uint32_t half = n_half; half >= 1; half >>= 1)
      run_threads(cdiv(n_half, 256), 256, [&] { k_ntt_dif_stage(d, tw.data(), n_half, half, n_half / half); });
  run_threads(cdiv(N, 256), 256, [&] { k_pointwise_mul(A.data(), B.data(), N, n_inv, 1); });
  for (uint32_t half = 1; half <= n_half; half <<= 1)
    run_threads(cdiv(n_half, 256), 256, [&] { k_ntt_dit_stage(A.data(), tw_inv.data(), n_half, half, n_half / half); });
  run_threads(cdiv(lo, 256), 256, [&] { k_poly_store(A.data(), lo, 0, 1, out.data()); });
  std::memcpy(out_std, out.data(), (size_t)lo * sizeof(Fr));
  return err;
}
}  // namespace

namespace {
// forward (dit = 0) or unscaled inverse (dit = 1) transform of 2^logn values: per-stage kernels vs the fused passes
int ntt_compare(const uint32_t* in_std, int logn, int dit, int max_k, uint32_t* out_stage, uint32_t* out_fused) {
  uint32_t N = 1u << logn, n_half = N >> 1;
  Fr root;
  for (int i = 0; i < 8; i++) root.l[i] = FrParams::ROOT(i);
  Fr w = root;
  for (int i = 0; i < FrParams::TWO_ADICITY - logn; i++) w = w.sqr();
  if (dit) w = w.inverse();
  std::vector<Fr> tw(n_half), A(N), B(N);
  std::memcpy(A.data(), in_std, (size_t)N * sizeof(Fr));
  B = A;
  run_threads(cdiv(n_half, 256), 256, [&] { k_twiddles(tw.data(), n_half, w); });
  if (!dit)
    for (uint32_t half = n_half; half >= 1; half >>= 1)
      run_threads(cdiv(n_half, 256), 256, [&] { k_ntt_dif_stage(A.data(), tw.data(), n_half, half, n_half / half); });
  else
    for (uint32_t half = 1; half <= n_half; half <<= 1)
      run_threads(cdiv(n_half, 256), 256, [&] { k_ntt_dit_stage(A.data(), tw.data(), n_half, half, n_half / half); });
  ntt_fused_passes(logn, dit, [&](uint32_t log_hbot, uint32_t k) {
    unsigned nb = N / kNttTile;
    for (unsigned b = 0; b < nb; b++) run_cta(b, 256, nb, [&] { k_ntt_fused(B.data(), tw.data(), n_half, log_hbot, k, dit); });
  }, max_k);
  std::memcpy(out_stage, A.data(), (size_t)N * sizeof(Fr));
  std::memcpy(out_fused, B.data(), (size_t)N * sizeof(Fr));
  return 0;
}
}  // namespace

template <class K> void stub_launch_threads(dim3 grid, unsigned nthreads, K k) { run_threads(grid, nthreads, k); }
template <class K> void stub_launch_cta(dim3 grid, unsigned nthreads, size_t smem, K k) {
  std::vector<uint8_t> shared(smem ? smem + 128 : 0);
  for (unsigned y = 0; y < grid.y; y++)
    for (unsigned b = 0; b < grid.x; b++) run_cta(b, nthreads, grid.x, k, y, grid.y, smem ? shared.data() : nullptr);
}

namespace {
// The library's OWN host orchestration (poly_host.cuh: transform plans, fused passes, division with the cached inverse
// series; qap_sparse.cuh: subproduct tree, Newton coefficients, divide and conquer) on the emulated kernels.
PolyCtx& poly_ctx() {
  static PolyCtx pc;
  return pc;
}
int qap_interpolate(const uint32_t* values_std, uint32_t n, uint32_t* coeffs_std) {
  size_t N = 1;
  while (N < n) N <<= 1;
  static std::map<size_t, std::unique_ptr<QapDomain>> doms;
  auto& dom = doms[N];
  if (!dom) {
    dom = std::make_unique<QapDomain>();
    if (qap_domain_build(poly_ctx(), *dom, N, nullptr)) return 1;
  }
  std::vector<Fr> v(n), c(N), out(n);
  std::memcpy(v.data(), values_std, (size_t)n * sizeof(Fr));
  for (auto& x : v) x = x.to_mont();
  QapWork wk;
  if (interpolate_ap(poly_ctx(), *dom, wk, v.data(), n, n, 1, c.data(), nullptr)) return 2;
  for (uint32_t i = 0; i < n; i++) out[i] = c[i].from_mont();
  for (size_t i = n; i < N; i++)
    if (!c[i].is_zero()) return 3;   // degree < n
  std::memcpy(coeffs_std, out.data(), (size_t)n * sizeof(Fr));
  return 0;
}
// h = DivisorPolynomial(a b - c, Z) straight from the values of a, b, c on {1..n} (qap_sparse.cuh: QapHDomain), as
// qap_h_enqueue runs it: the values of c are overwritten by the products a_j b_j, so any c gives the same quotient
int qap_h_direct(const uint32_t* abc_std, uint32_t n, uint32_t* h_std) {
  size_t N = 1;
  while (N < n) N <<= 1;
  QapDomain dom;
  if (qap_domain_build(poly_ctx(), dom, N, nullptr)) return 1;
  std::vector<Fr> v(3 * (size_t)n), d(3 * N);
  std::memcpy(v.data(), abc_std, v.size() * sizeof(Fr));
  for (auto& x : v) x = x.to_mont();
  QapWork wk;
  QapHDomain hd;
  if (qap_hdomain_build(poly_ctx(), hd, n, nullptr)) return 3;
  if (qap_h_from_values(poly_ctx(), dom, wk, hd, v.data(), d.data(), nullptr)) return 4;
  const Fr* c = hd.coef.as<Fr>();
  for (uint32_t i = 0; i + 1 < n; i++) {
    Fr x = c[i].from_mont();
    std::memcpy(h_std + 8 * (size_t)i, &x, sizeof(Fr));
  }
  for (size_t i = n - 1; i < hd.tree.N; i++)
    if (!c[i].is_zero()) return 5;   // degree <= n - 2
  return 0;
}
int qap_zero_poly(uint32_t n, uint32_t* out_std) {   // prod_{i=1..n}(x - i): Newton basis element n
  size_t N = 1;
  while (N < (size_t)n + 1) N <<= 1;
  QapDomain dom;
  if (qap_domain_build(poly_ctx(), dom, N, nullptr)) return 1;
  std::vector<Fr> P(N, Fr::zero()), X(N);
  P[n] = Fr::one();
  if (newton_to_monomial(poly_ctx(), dom, P.data(), X.data(), 1, nullptr)) return 2;
  for (uint32_t i = 0; i <= n; i++) {
    Fr v = P[i].from_mont();
    std::memcpy(out_std + 8 * (size_t)i, &v, sizeof(Fr));
  }
  return 0;
}
int poly_div_orch(const uint32_t* a_std, uint32_t na, const uint32_t* b_std, uint32_t nb, uint32_t* q_std, uint32_t* rem_std) {
  Divisor dv;
  std::vector<Fr> b(nb), a(na), q(na - nb + 1), rem(nb > 1 ? nb - 1 : 1);
  std::memcpy(b.data(), b_std, (size_t)nb * sizeof(Fr));
  std::memcpy(a.data(), a_std, (size_t)na * sizeof(Fr));
  for (auto& x : b) x = x.to_mont();
  if (dv.b_mont.alloc(nb * sizeof(Fr))) return 1;
  std::memcpy(dv.b_mont.p, b.data(), nb * sizeof(Fr));
  dv.nb = nb;
  int err = 0;
  if (poly_div_device(poly_ctx(), dv, a.data(), na, 0, q.data(), rem_std ? rem.data() : nullptr, &err, nullptr)) return 2;
  std::memcpy(q_std, q.data(), q.size() * sizeof(Fr));
  if (rem_std && nb > 1) std::memcpy(rem_std, rem.data(), (size_t)(nb - 1) * sizeof(Fr));
  return err ? 100 + err : 0;
}
}  // namespace

extern "C" {
int t_qap_interpolate(const uint32_t* values_std, uint32_t n, uint32_t* coeffs_std) { return qap_interpolate(values_std, n, coeffs_std); }
int t_qap_zero_poly(uint32_t n, uint32_t* out_std) { return qap_zero_poly(n, out_std); }
int t_qap_h_direct(const uint32_t* abc_std, uint32_t n, uint32_t* h_std) { return qap_h_direct(abc_std, n, h_std); }
int t_poly_div_orch(const uint32_t* a, uint32_t na, const uint32_t* b, uint32_t nb, uint32_t* q, uint32_t* rem) {
  return poly_div_orch(a, na, b, nb, q, rem);
}
int t_ntt_compare(const uint32_t* in_std, int logn, int dit, int max_k, uint32_t* out_stage, uint32_t* out_fused) {
  return ntt_compare(in_std, logn, dit, max_k, out_stage, out_fused);
}
int t_poly_mul_kernels(const uint32_t* a, uint32_t la, const uint32_t* b, uint32_t lb, uint32_t* out) {
  return poly_mul_kernels(a, la, b, lb, out);
}
// sum_i scalars[i] * P_i through the library's MSM engine; S = 0: XYZZ accumulation, else batched-affine slices of S
int t_msm_full(int group, const uint32_t* jac_std, const uint32_t* scalars_std, uint32_t n, uint32_t c, uint32_t S, uint32_t* out_std) {
  return group == 1 ? msm_full<Fq>(group, jac_std, scalars_std, n, c, S, out_std)
                    : msm_full<Fq2>(group, jac_std, scalars_std, n, c, S, out_std);
}
// glv.cuh on a 32-thread emulated warp: lanes 0..15 compute k0 * P0, lanes 16..31 k1 * P1 — the two half-warps of
// k_groth16_products / k_ic_terms — with the scalars split by glv_decompose exactly as the host side of the library does.
// pts: two Jacobian points (X, Y, Z standard form, 24 words each); ks: two scalars (standard form, < r); out: two Jacobian
// points, standard form.  Returns glv_decompose's status.
int t_glv_mul(const uint32_t* pts, const uint32_t* ks, uint32_t* out) {
  GlvScalars g;
  Jacobian<Fq> p[2], res[2];
  for (int i = 0; i < 2; i++) {
    Fr k;
    std::memcpy(&k, ks + 8 * i, sizeof(Fr));
    if (glv_decompose(k, g.k[i], g.neg[i])) return 1;
    p[i] = Jacobian<Fq>{load_std<Fq>(pts + 24 * i), load_std<Fq>(pts + 24 * i + 8), load_std<Fq>(pts + 24 * i + 16)};
  }
  run_cta(0, 32, 1, [&] {
    const uint32_t t = threadIdx.x & 31u, grp = t >> 4;
    Jacobian<Fq> r = glv_mul_halfwarp(p[grp], g.k[grp], g.neg[grp], t);
    if ((t & 15u) == 0) res[grp] = r;
  });
  for (int i = 0; i < 2; i++) {
    store_std(out + 24 * i, res[i].X);
    store_std(out + 24 * i + 8, res[i].Y);
    store_std(out + 24 * i + 16, res[i].Z);
  }
  return 0;
}
// One-warp-per-pairing code (pairing_warp.cuh) on a 32-thread emulated warp.  g1 = (x, y), g2 = (x.c0, x.c1, y.c0, y.c1), affine
// standard form; out = 12 field elements in the reference's [2][3][2] order.  mode 0: the whole pairing; mode 1: only an
// F_q^12 product of in (12 elements) with in2 -> out (the tower product against f12_mul is checked by the caller).
// Returns the number of coefficient mismatches against the thread-per-pairing restatement of pairing.cuh.
int t_pairing_warp(const uint32_t* g1, const uint32_t* g2, uint32_t* out) {
  F2::B px = load_std<F2::B>(g1), py = load_std<F2::B>(g1 + 8);
  F2 qx = load_std<F2>(g2), qy = load_std<F2>(g2 + 16);
  static wp::Ws ws;
  run_cta(0, 32, 1, [&] { wp::pairing(ws, px, py, qx, qy); });
  F12 ref = pairing_affine_t<true>(px, py, qx, qy);
  const F2* parts[6] = {&ref.a.a, &ref.a.b, &ref.a.c, &ref.b.a, &ref.b.b, &ref.b.c};
  int bad = 0;
  for (int k = 0; k < 6; k++) {
    if (!(ws.r[wp::RF][k] == *parts[k])) bad++;
    store_std(out + 16 * k, ws.r[wp::RF][k]);
  }
  return bad;
}
int t_f12_warp_ops(const uint32_t* a_std, const uint32_t* b_std, uint32_t* out_mul, uint32_t* out_frob2, uint32_t* out_expu_conj) {
  static wp::Ws ws;
  F12 x, y;
  F2* xs[6] = {&x.a.a, &x.a.b, &x.a.c, &x.b.a, &x.b.b, &x.b.c};
  F2* ys[6] = {&y.a.a, &y.a.b, &y.a.c, &y.b.a, &y.b.b, &y.b.c};
  for (int k = 0; k < 6; k++) {
    *xs[k] = load_std<F2>(a_std + 16 * k);
    *ys[k] = load_std<F2>(b_std + 16 * k);
    ws.r[2][k] = *xs[k];
    ws.r[3][k] = *ys[k];
  }
  F2 qd = F2::one();
  run_cta(0, 32, 1, [&] {
    wp::pairing_constants(ws);
    wp::f12_mul(ws, 4, 2, 3);
    wp::f12_frobenius(ws, 5, 2, 2);
    wp::f12_exp_u(ws, 6, 2);
    wp::f12_conj(ws, 6, 6);
    wp::f12_mul(ws, 2, 2, 2);      // aliased square
    wp::f12_inverse(ws, 7, 3);
    wp::f12_frobenius(ws, 8, 3, 1);
    wp::f12_frobenius(ws, 9, 3, 3);
  });
  (void)qd;
  auto cmp = [&](int reg, const F12& r) {
    const F2* parts[6] = {&r.a.a, &r.a.b, &r.a.c, &r.b.a, &r.b.b, &r.b.c};
    int bad = 0;
    for (int k = 0; k < 6; k++) bad += !(ws.r[reg][k] == *parts[k]);
    return bad;
  };
  int bad = cmp(4, f12_mul(x, y)) + 10 * cmp(5, f12_frobenius<2>(x)) + 100 * cmp(6, f12_conj(f12_exp_u(x))) + 1000 * cmp(2, f12_sqr(x)) +
            10000 * cmp(7, f12_inverse(y)) + 100000 * cmp(8, f12_frobenius<1>(y)) + 1000000 * cmp(9, f12_frobenius<3>(y));
  for (int k = 0; k < 6; k++) {
    store_std(out_mul + 16 * k, ws.r[4][k]);
    store_std(out_frob2 + 16 * k, ws.r[5][k]);
    store_std(out_expu_conj + 16 * k, ws.r[6][k]);
  }
  return bad;
}
int t_msm_tail(int group, const uint32_t* slice_pts_std, const uint32_t* slice_off, uint32_t nbuckets, uint32_t seg, uint32_t* out_std) {
  return group == 1 ? msm_tail<Fq>(slice_pts_std, slice_off, nbuckets, seg, out_std)
                    : msm_tail<Fq2>(slice_pts_std, slice_off, nbuckets, seg, out_std);
}
// group: 1 = G1 (F_q), 2 = G2 (F_q^2); variant: 0 product backward kernel, 1 _lr, 2 _sp, 3 prefetch variant; T in {8, 32}
// fwd_variant: -1 = host restatement of the forward pass; 0 / 1 / 2 = run the forward KERNEL (product, prefetch, _sp)
// CTA by CTA and compare its pre / others / btot with the restatement (return code 10+r, 20+r, 30+r on a mismatch in round r)
int t_affine_rounds(int group, int variant, int fwd_variant, int T, const uint32_t* table_std, uint32_t n_pts, const uint32_t* entries,
                    const uint32_t* slice_start, const uint32_t* slice_end, uint32_t nslices, uint32_t R, uint32_t* out_std) {
  if (group == 1 && T == 8) return affine_rounds<Fq, 8>(variant, fwd_variant, table_std, n_pts, entries, slice_start, slice_end, nslices, R, out_std);
  if (group == 1 && T == 32) return affine_rounds<Fq, 32>(variant, fwd_variant, table_std, n_pts, entries, slice_start, slice_end, nslices, R, out_std);
  if (group == 2 && T == 8) return affine_rounds<Fq2, 8>(variant, fwd_variant, table_std, n_pts, entries, slice_start, slice_end, nslices, R, out_std);
  return -1;
}
}
