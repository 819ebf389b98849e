// Bucket accumulation by BATCHED AFFINE ADDITION (the default hot path for large MSMs).
//
// An affine addition costs 1 inversion + 2M + 1S; with Montgomery's trick a batch
// of denominators shares one inversion at 3M each, so a bucket add costs ~6.5 field
// multiplications instead of the 10 (8M + 2S) of the XYZZ mixed add — and the
// integer multiply pipe (IMAD.WIDE) is what bounds this kernel
// (DESIGN.md §4).
//
// Shape.  Buckets are cut into slices of exactly S = 2^R leaf slots (the tail of a
// bucket is padded with the point at infinity), so every slice is a perfect
// binary tree: round r (1..R) has S >> r independent pair additions per slice and
// pair p of the whole MSM is (slice p / q, position p % q), q = S >> r — no
// ragged bookkeeping.  Each round is three launches:
//   k_affine_forward   thread t walks its T pairs, recomputes each denominator
//                      d = x2 - x1 (2y for a doubling, 1 for the infinity cases),
//                      stores the running prefix product, and a block-wide
//                      shuffle/shared-memory scan gives every thread the product
//                      of all OTHER threads' totals; the block total goes to HBM
//   k_affine_invert    one inversion per block total (a few thousand per round —
//                      negligible work, pure latency: binary Euclid, a warp each)
//   k_affine_backward  thread t derives 1/total_t, walks its pairs backwards
//                      peeling 1/d off the running inverse, and writes the sums
// After R rounds every slice is one affine point; k_merge_slices_affine folds the
// slices of a bucket into the XYZZ bucket array consumed by the weighted reduction.
// Measured and dropped: register-staged and L2-prefetch software pipelines of the operand
// fetches, an inlined multiply, a backward pass ordered for short live ranges, a thread-per-slice variant with the
// rounds fused, fewer pairs per thread in the late rounds, an XYZZ tail after a few affine rounds.
#pragma once
#include "msm.cuh"

namespace b200 {

constexpr int kAffBlock = 128;    // threads per block
constexpr int kAffPairs = 32;     // pairs per thread per round

// Tree nodes of a round, x- and y-coordinates in SEPARATE arrays: the forward pass of the next round needs only the two
// x-coordinates of a pair — 64 (G1) / 128 (G2) contiguous bytes here instead of two whole points — and the backward pass
// reads / writes the same bytes either way.  (The window-precomputed CRS table stays point-interleaved: its gathers are
// random, and a 64-byte point is one DRAM access.)
template <class F>
struct NodeBuf {
  F* x;
  F* y;
};

template <class F>
struct AffineRound {
  const Affine<F>* table;     // precomputed points (round 1 leaves)
  const uint32_t* entries;    // sorted entry ids (round 1)
  const uint32_t* slice_start;
  const uint32_t* slice_end;
  const uint32_t* nslices_ptr;  // device: slice_off[m]
  NodeBuf<F> prev;            // nodes of the previous round (r > 1): nslices * 2q
  NodeBuf<F> out;             // nodes of this round: nslices * q
  F* pre;                     // prefix products, one per pair
  F* others;                  // per thread: product of the other threads' totals in its block
  F* btot;                    // per block: product of all denominators (then inverted in place)
  uint2* pair_ids;            // round 1: (entry id of P, entry id of Q) per pair, 0xffffffff = absent (forward writes, backward reads)
  uint32_t q_log;             // log2(pairs per slice in this round)
  uint32_t round;             // 1-based
};

// operands of pair `p`; returns false when p is beyond the live range
template <class F>
__device__ __forceinline__ bool aff_operands(const AffineRound<F>& a, uint32_t p, uint32_t npairs, Affine<F>& P, Affine<F>& Q) {
  if (p >= npairs) return false;
  uint32_t slice = p >> a.q_log, j = p & ((1u << a.q_log) - 1u);
  if (a.round == 1) {
    uint32_t s = a.slice_start[slice], e = a.slice_end[slice];
    uint32_t i0 = s + 2 * j, i1 = i0 + 1;
    P = Affine<F>::inf();
    Q = Affine<F>::inf();
    if (i0 < e) {
      uint32_t en = a.entries[i0];
      P = ld_affine_gather(&a.table[en >> 1]);
      if ((en & 1) && !P.is_inf()) P.y = P.y.neg();
    }
    if (i1 < e) {
      uint32_t en = a.entries[i1];
      Q = ld_affine_gather(&a.table[en >> 1]);
      if ((en & 1) && !Q.is_inf()) Q.y = Q.y.neg();
    }
  } else {
    size_t base = ((size_t)slice << (a.q_log + 1)) + 2 * j;
    P = Affine<F>{ld_fe(&a.prev.x[base]), ld_fe(&a.prev.y[base])};
    Q = Affine<F>{ld_fe(&a.prev.x[base + 1]), ld_fe(&a.prev.y[base + 1])};
  }
  return true;
}

// kind of the addition and its denominator (never zero)
//   0: P or Q at infinity / P = -Q  -> d = 1 ;  1: generic, d = x2 - x1 ;  2: doubling, d = 2 y1
template <class F>
__device__ __forceinline__ int aff_denominator(const Affine<F>& P, const Affine<F>& Q, F& d) {
  if (P.is_inf() || Q.is_inf()) {
    d = F::one();
    return 0;
  }
  F dx = Q.x - P.x;
  if (!dx.is_zero()) {
    d = dx;
    return 1;
  }
  if (P.y == Q.y && !P.y.is_zero()) {
    d = P.y.dbl();
    return 2;
  }
  d = F::one();
  return 0;
}

// x-coordinate only, for the forward pass (a G2 point is a full 128-byte line: its x is half of it)
template <class P, bool I>
__device__ __forceinline__ Fp<P, I> ld_x_gather(const Affine<Fp<P, I>>* p) { Fp<P, I> r; ld256_g64(&p->x, r.l); return r; }
template <bool I>
__device__ __forceinline__ Fq2T<I> ld_x_gather(const Affine<Fq2T<I>>* p) { return ld_fe(&p->x); }

// Denominator of pair `p` for the forward pass.  The generic case needs only the two x-coordinates, so only those
// are fetched (half the registers and load instructions of the full operands -> the forward kernel runs at twice the
// occupancy, which is what hides its dependent index -> point gathers); whenever an x is zero (infinity) or the x's
// coincide (doubling / P = -Q) the full operands decide, exactly as in the backward pass.
template <class F>
__device__ __forceinline__ bool aff_forward_denominator(const AffineRound<F>& a, uint32_t p, uint32_t npairs, F& d) {
  if (p >= npairs) return false;
  uint32_t slice = p >> a.q_log, j = p & ((1u << a.q_log) - 1u);
  F x1, x2;
  if (a.round == 1) {
    uint32_t s = a.slice_start[slice], e = a.slice_end[slice];
    uint32_t i0 = s + 2 * j, i1 = i0 + 1;
    if (i1 >= e) {  // at most one live operand: nothing to invert
      if (a.pair_ids) a.pair_ids[p] = make_uint2(i0 < e ? a.entries[i0] : 0xffffffffu, 0xffffffffu);
      d = F::one();
      return true;
    }
    uint32_t e0 = a.entries[i0], e1 = a.entries[i1];
    if (a.pair_ids) a.pair_ids[p] = make_uint2(e0, e1);
    x1 = ld_x_gather(&a.table[e0 >> 1]);
    x2 = ld_x_gather(&a.table[e1 >> 1]);
  } else {
    size_t base = ((size_t)slice << (a.q_log + 1)) + 2 * j;
    x1 = ld_fe(&a.prev.x[base]);
    x2 = ld_fe(&a.prev.x[base + 1]);
  }
  F dx = x2 - x1;
  if (x1.is_zero() || x2.is_zero() || dx.is_zero()) {
    Affine<F> P, Q;
    aff_operands(a, p, npairs, P, Q);
    aff_denominator(P, Q, d);
  } else {
    d = dx;
  }
  return true;
}

template <class F>
__device__ __forceinline__ F shfl_up_fe(const F& v, int delta) {
  F r;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&v);
  uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int i = 0; i < (int)(sizeof(F) / 4); i++) d[i] = __shfl_up_sync(0xffffffffu, s[i], delta);
  return r;
}
template <class F>
__device__ __forceinline__ F shfl_down_fe(const F& v, int delta) {
  F r;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&v);
  uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int i = 0; i < (int)(sizeof(F) / 4); i++) d[i] = __shfl_down_sync(0xffffffffu, s[i], delta);
  return r;
}
template <class F>
__device__ __forceinline__ F shfl_idx_fe(const F& v, int lane) {
  F r;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&v);
  uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int i = 0; i < (int)(sizeof(F) / 4); i++) d[i] = __shfl_sync(0xffffffffu, s[i], lane);
  return r;
}

template <class F, int kAffT, int MINB = 1>
__global__ void __launch_bounds__(kAffBlock, MINB) k_affine_forward(AffineRound<F> a) {
  __shared__ F wtot[kAffBlock / 32];
  const uint32_t nslices = *a.nslices_ptr;
  const uint32_t npairs = nslices << a.q_log;
  const uint32_t block_base = blockIdx.x * (kAffBlock * kAffT);
  if (block_base >= npairs) {  // whole block idle (grid sized for the worst case)
    if (threadIdx.x == 0) a.btot[blockIdx.x] = F::one();
    return;
  }
  const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
  F run = F::one();
  for (int k = 0; k < kAffT; k++) {
    uint32_t p = block_base + k * kAffBlock + t;  // block-interleaved: coalesced across the warp
    F d;
    if (aff_forward_denominator(a, p, npairs, d)) {
      a.pre[p] = run;
      run = run * d;
    }
  }
  // Every thread needs the product of all OTHER threads' totals of the block (no division available):
  // inclusive prefix and suffix scans over the warp's lanes, shifted by one, times the other warps' totals.
  F incl = run;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    F up = shfl_up_fe(incl, off);
    if ((int)lane >= off) incl = incl * up;
  }
  F sincl = run;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    F dn = shfl_down_fe(sincl, off);
    if ((int)lane + off < 32) sincl = sincl * dn;
  }
  F pex = shfl_up_fe(incl, 1), sex = shfl_down_fe(sincl, 1);
  if (lane == 0) pex = F::one();
  if (lane == 31) sex = F::one();
  F warp_total = shfl_idx_fe(incl, 31);
  if (lane == 0) wtot[warp] = warp_total;
  __syncthreads();
  F other_warps = F::one();
#pragma unroll
  for (int w = 0; w < kAffBlock / 32; w++)
    if (w != (int)warp) other_warps = other_warps * wtot[w];
  uint32_t gthread = blockIdx.x * kAffBlock + t;
  a.others[gthread] = pex * sex * other_warps;
  if (t == 0) a.btot[blockIdx.x] = other_warps * wtot[0];
}

// One warp per block total, lane 0 working: the binary-Euclid inversion has data-dependent control flow, and this
// launch is pure latency (a few thousand inversions between two machine-filling passes), far longer with a^(p-2).
template <class F>
__global__ void __launch_bounds__(128) k_affine_invert(F* btot, uint32_t nblocks_live) {
  uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if ((threadIdx.x & 31u) || i >= nblocks_live) return;
  btot[i] = btot[i].inverse_vartime();
}

template <class F, int kAffT, int MINB = 1>
__global__ void __launch_bounds__(kAffBlock, MINB) k_affine_backward(AffineRound<F> a) {
  const uint32_t nslices = *a.nslices_ptr;
  const uint32_t npairs = nslices << a.q_log;
  const uint32_t block_base = blockIdx.x * (kAffBlock * kAffT);
  if (block_base >= npairs) return;
  const uint32_t t = threadIdx.x;
  uint32_t gthread = blockIdx.x * kAffBlock + t;
  F inv_run = a.btot[blockIdx.x] * a.others[gthread];  // 1 / (product of this thread's denominators)
  for (int k = kAffT - 1; k >= 0; k--) {
    uint32_t p = block_base + k * kAffBlock + t;
    Affine<F> P, Q;
    if (!aff_operands(a, p, npairs, P, Q)) continue;
    F d;
    int kind = aff_denominator(P, Q, d);
    F inv_d = inv_run * a.pre[p];
    inv_run = inv_run * d;
    Affine<F> Rr;
    if (kind == 1) {
      F lam = (Q.y - P.y) * inv_d;
      F x3 = lam.sqr() - P.x - Q.x;
      Rr = Affine<F>{x3, lam * (P.x - x3) - P.y};
    } else if (kind == 2) {
      F xx = P.x.sqr();
      F lam = (xx.dbl() + xx) * inv_d;
      F x3 = lam.sqr() - P.x.dbl();
      Rr = Affine<F>{x3, lam * (P.x - x3) - P.y};
    } else {
      Rr = P.is_inf() ? Q : (Q.is_inf() ? P : Affine<F>::inf());
    }
    a.out.x[p] = Rr.x;
    a.out.y[p] = Rr.y;
  }
}

// ---- staged backward pass: TMA bulk copies + mbarrier (rounds >= 2), cp.async gathers (round 1) ---------------
// The backward pass is bound by the integer-multiply pipe, but a third of its stall samples are long-scoreboard
// waits: every iteration starts with the operand fetch (round 1: two random 64/128-byte point gathers from a >= 1 GB
// table; later rounds: the node pair of the previous round) plus the prefix product, all through registers.  Here the
// operands of the NEXT pair are staged into shared memory while the multiplies of the current pair run, without
// holding a single register across the fetch:
//   rounds >= 2  the 32 node pairs of a warp's iteration are CONTIGUOUS (4 / 8 KB) and so are its 32 prefix products:
//                lane 0 issues two TMA bulk copies (cp.async.bulk.shared.global, SASS UBLKCP — a warp-uniform
//                instruction, which is why one lane issues for the warp) that complete_tx on the warp's mbarrier,
//                armed with arrive.expect_tx; all lanes then wait on its phase parity;
//   round 1      the operands are per-thread random gathers: each thread copies its two points and its prefix product
//                with 16-byte cp.async (LDGSTS) into its own row and waits on its own cp.async group.  The entry ids are
//                needed one step earlier: the forward pass leaves them in `pair_ids` (8 B per pair, coalesced).
// The copies for pair k-1 are issued in the MIDDLE of pair k, right after the last use of pair k's row, and have three
// field multiplications of time to land.  Rows are read back with 128-bit shared loads; the linear row layout the bulk
// copy produces costs bank conflicts on them (8-way on the points), ~300 extra shared-pipe cycles against ~20 000 cycles
// of arithmetic per warp iteration.
constexpr uint32_t kNoEntry = 0xffffffffu;
template <class F>
struct AffStageLayout {
  static constexpr uint32_t kPairBytes = 2 * sizeof(Affine<F>);                        // 128 B (G1) / 256 B (G2)
  // per thread: [P.x | Q.x] in the X region, [P.y | Q.y] in the Y region (the node arrays are x / y separated), one prefix product
  static constexpr uint32_t kX = 0, kY = kAffBlock * 2 * sizeof(F), kPre = kAffBlock * kPairBytes, kBar = kPre + kAffBlock * sizeof(F);
  static constexpr uint32_t kSmem = kBar + (kAffBlock / 32) * 8;                       // 20.5 KB (G1) / 41 KB (G2)
};

namespace tma {
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__cvta_generic_to_shared(p);
#else
  return (uint32_t)(uintptr_t)p;
#endif
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
#ifdef __CUDA_ARCH__
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#else
  (void)bar; (void)count;
#endif
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
#ifdef __CUDA_ARCH__
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
#else
  (void)bar; (void)bytes;
#endif
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#ifdef __CUDA_ARCH__
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
#elif !defined(__CUDACC__)   // CPU test vehicle: the leader's copy was synchronous; a warp barrier orders it before the followers' reads
  (void)bar; (void)parity;
  stub_syncwarp();
#endif
}
// global -> shared bulk copy (TMA, SASS: UBLKCP); bytes a multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
#else   // CPU test vehicle: synchronous copy, the barrier is a no-op
  (void)bar;
  memcpy(dst_smem, src_gmem, bytes);
#endif
}
// per-thread asynchronous 16-byte copies (LDGSTS), L2 only; BYTES a multiple of 16
template <int BYTES>
__device__ __forceinline__ void cp_async(void* dst_smem, const void* src_gmem) {
#ifdef __CUDA_ARCH__
#pragma unroll
  for (int o = 0; o < BYTES; o += 16)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem) + o), "l"(static_cast<const char*>(src_gmem) + o)
                 : "memory");
#else
  memcpy(dst_smem, src_gmem, BYTES);
#endif
}
__device__ __forceinline__ void cp_async_commit_and_wait() {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
#endif
}
__device__ __forceinline__ void cp_async_commit() {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void cp_async_wait() {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.wait_group 0;" ::: "memory");
#endif
}
__device__ __forceinline__ void lds128(const void* p, uint32_t* o) {
#ifdef __CUDA_ARCH__
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(o[0]), "=r"(o[1]), "=r"(o[2]), "=r"(o[3]) : "r"(smem_u32(p)));
#else
  memcpy(o, p, 16);
#endif
}
template <class P, bool I>
__device__ __forceinline__ Fp<P, I> ld_row(const uint8_t* p, Fp<P, I>*) {
  Fp<P, I> r;
  lds128(p, r.l);
  lds128(p + 16, r.l + 4);
  return r;
}
template <bool I>
__device__ __forceinline__ Fq2T<I> ld_row(const uint8_t* p, Fq2T<I>*) {
  Fq2T<I> r;
  r.c0 = ld_row(p, (decltype(r.c0)*)nullptr);
  r.c1 = ld_row(p + 32, (decltype(r.c1)*)nullptr);
  return r;
}
__device__ __forceinline__ void syncwarp() {
#ifdef __CUDA_ARCH__
  __syncwarp();
#elif !defined(__CUDACC__)
  stub_syncwarp();
#endif
}
}  // namespace tma

#ifndef __CUDACC__
inline thread_local uint8_t* g_stub_dyn_smem = nullptr;   // CPU test vehicle: the emulated CTA's dynamic shared memory
#endif

template <class F, int kAffT, int MINB = 1>
__global__ void __launch_bounds__(kAffBlock, MINB) k_affine_backward_staged(AffineRound<F> a) {
  using L = AffStageLayout<F>;
#ifdef __CUDACC__
  extern __shared__ __align__(128) uint8_t aff_smem[];
  uint8_t* smem = aff_smem;
#else
  uint8_t* smem = g_stub_dyn_smem;
#endif
  const uint32_t nslices = *a.nslices_ptr;
  const uint32_t npairs = nslices << a.q_log;
  const uint32_t block_base = blockIdx.x * (kAffBlock * kAffT);
  if (block_base >= npairs) return;
  const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
  uint8_t* row_x = smem + L::kX + (size_t)t * 2 * sizeof(F);
  uint8_t* row_y = smem + L::kY + (size_t)t * 2 * sizeof(F);
  uint8_t* row_pre = smem + L::kPre + (size_t)t * sizeof(F);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + L::kBar) + warp;
  const bool leaves = a.round == 1;
  if (!leaves && lane == 0) tma::mbar_init(bar, 1);
  tma::syncwarp();

  // stage the operands of pair p (this thread's pair of the warp-iteration starting at pair p0 = p - lane)
  auto issue = [&](uint32_t p, uint2 ids) {
    if (leaves) {   // per-thread gathers
      if (p < npairs) {
        if (ids.x != kNoEntry) {
          tma::cp_async<(int)sizeof(F)>(row_x, &a.table[ids.x >> 1].x);
          tma::cp_async<(int)sizeof(F)>(row_y, &a.table[ids.x >> 1].y);
        }
        if (ids.y != kNoEntry) {
          tma::cp_async<(int)sizeof(F)>(row_x + sizeof(F), &a.table[ids.y >> 1].x);
          tma::cp_async<(int)sizeof(F)>(row_y + sizeof(F), &a.table[ids.y >> 1].y);
        }
        tma::cp_async<(int)sizeof(F)>(row_pre, &a.pre[p]);
      }
      tma::cp_async_commit();
    } else if (lane == 0) {   // one lane per warp: three bulk copies for the warp's 32 contiguous pairs (x's, y's, prefix products)
      uint32_t valid = p < npairs ? (npairs - p < 32u ? npairs - p : 32u) : 0u;
      tma::mbar_arrive_expect_tx(bar, valid * (L::kPairBytes + (uint32_t)sizeof(F)));
      if (valid) {
        tma::bulk_g2s(row_x, &a.prev.x[2 * (size_t)p], valid * 2 * (uint32_t)sizeof(F), bar);
        tma::bulk_g2s(row_y, &a.prev.y[2 * (size_t)p], valid * 2 * (uint32_t)sizeof(F), bar);
        tma::bulk_g2s(row_pre, &a.pre[p], valid * (uint32_t)sizeof(F), bar);
      }
    }
  };
  auto ids_of = [&](uint32_t p) -> uint2 {
    if (leaves && p < npairs) return a.pair_ids[p];
    return make_uint2(0u, 0u);
  };

  uint32_t gthread = blockIdx.x * kAffBlock + t;
  F inv_run = a.btot[blockIdx.x] * a.others[gthread];  // 1 / (product of this thread's denominators)
  uint2 ids_cur = ids_of(block_base + (kAffT - 1) * kAffBlock + t);
  issue(block_base + (kAffT - 1) * kAffBlock + t, ids_cur);
  uint32_t phase = 0;
  for (int k = kAffT - 1; k >= 0; k--) {
    const uint32_t p = block_base + k * kAffBlock + t;
    uint2 ids_next = make_uint2(0u, 0u);
    if (k > 0) ids_next = ids_of(p - kAffBlock);          // coalesced; consumed in the middle of this iteration
    if (leaves) tma::cp_async_wait();
    else tma::mbar_wait(bar, phase);
    phase ^= 1u;
    const bool live = p < npairs;
    Affine<F> P = Affine<F>::inf(), Q = Affine<F>::inf();
    F pre = F::one(), d = F::one();
    int kind = 0;
    if (live) {
      const bool has_p = !leaves || ids_cur.x != kNoEntry, has_q = !leaves || ids_cur.y != kNoEntry;
      if (has_p) {
        P.x = tma::ld_row(row_x, (F*)nullptr);
        P.y = tma::ld_row(row_y, (F*)nullptr);
        if (leaves && (ids_cur.x & 1) && !P.is_inf()) P.y = P.y.neg();
      }
      if (has_q) {
        Q.x = tma::ld_row(row_x + sizeof(F), (F*)nullptr);
        Q.y = tma::ld_row(row_y + sizeof(F), (F*)nullptr);
        if (leaves && (ids_cur.y & 1) && !Q.is_inf()) Q.y = Q.y.neg();
      }
      pre = tma::ld_row(row_pre, (F*)nullptr);
      kind = aff_denominator(P, Q, d);
    }
    F inv_d = inv_run * pre;
    if (live) inv_run = inv_run * d;
    // every value of this iteration's rows has been consumed (compared or multiplied) by every lane: refill them
    tma::syncwarp();
    if (k > 0) issue(p - kAffBlock, ids_next);
    ids_cur = ids_next;
    if (!live) continue;
    Affine<F> Rr;
    if (kind == 1) {
      F lam = (Q.y - P.y) * inv_d;
      F x3 = lam.sqr() - P.x - Q.x;
      Rr = Affine<F>{x3, lam * (P.x - x3) - P.y};
    } else if (kind == 2) {
      F xx = P.x.sqr();
      F lam = (xx.dbl() + xx) * inv_d;
      F x3 = lam.sqr() - P.x.dbl();
      Rr = Affine<F>{x3, lam * (P.x - x3) - P.y};
    } else {
      Rr = P.is_inf() ? Q : (Q.is_inf() ? P : Affine<F>::inf());
    }
    a.out.x[p] = Rr.x;
    a.out.y[p] = Rr.y;
  }
}

// buckets[b-1] = sum of the (affine) slice results of bucket b.
// A thread folds up to kMergeSeq slices itself; only buckets beyond that (skewed scalar distributions) take the warp path.
// bases_create picks S so that the MEAN bucket holds 6..12 slices, and the population spreads around it: with the bound at 12
// (rounds 1-2 of this kernel) nearly half the buckets of a set whose mean sat just under 12 slices went down the warp path,
// one after the other, so a G1 MSM just below the next S was far slower than one just above it (tools/slice_cliff.py).  Twice the largest mean leaves the warp path to the genuinely skewed buckets.
constexpr uint32_t kMergeSeq = 24;
template <class F>
__global__ void __launch_bounds__(128)
k_merge_slices_affine(NodeBuf<F> slice_pts, SliceTables st, uint32_t nbuckets,
                      XYZZ<F>* __restrict__ buckets) {
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x + 1;
  uint32_t lane = threadIdx.x & 31;
  uint32_t first = 0, cnt = 0;
  if (b <= nbuckets) {
    first = st.slice_off[b];
    cnt = st.slice_off[b + 1] - first;
    if (cnt <= kMergeSeq) {  // the common case: a handful of slices per bucket
      XYZZ<F> acc = XYZZ<F>::inf();
      for (uint32_t k = 0; k < cnt; k++) xyzz_madd(acc, Affine<F>{ld_fe(&slice_pts.x[first + k]), ld_fe(&slice_pts.y[first + k])});
      buckets[b - 1] = acc;
    }
  }
  uint32_t multi = __ballot_sync(0xffffffffu, cnt > kMergeSeq);  // skewed buckets: the whole warp sums them
  while (multi) {
    int j = __ffs(multi) - 1;
    multi &= multi - 1;
    uint32_t f = __shfl_sync(0xffffffffu, first, j), c = __shfl_sync(0xffffffffu, cnt, j);
    uint32_t bj = __shfl_sync(0xffffffffu, b, j);
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t k = lane; k < c; k += 32) xyzz_madd(acc, Affine<F>{ld_fe(&slice_pts.x[f + k]), ld_fe(&slice_pts.y[f + k])});
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      XYZZ<F> other = shfl_down_struct(acc, off, 32);
      xyzz_add(acc, other);
    }
    if (lane == 0) buckets[bj - 1] = acc;
  }
}

}  // namespace b200
