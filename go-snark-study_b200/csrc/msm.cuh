// Pippenger multi-scalar multiplication over a device-resident, window-
// precomputed base set.  Replaces the reference's per-term double-and-add loops
// (groth16/groth16.go:243-250,269-271; snark.go:265-286).
//
// Data layout in HBM (DESIGN.md §3):
//   table   [t][n]     Affine<F>, Montgomery form: table[j][i] = 2^(c*j) * P_i
//                      (64 B per G1 point, 128 B per G2 point, 32 B-aligned so a
//                      point is 4 / 8 sector-exact 128-bit loads)
//   scalars [n]        4 x u64 standard form (or Montgomery if produced by the
//                      NTT pipeline)
//   entries [nwin*n]   u32: (j*n + i) << 1 | sign, counting-sorted by bucket
//   buckets [k*G*B]    XYZZ<F>, B = 2^(c-1) (signed digits) per window group of each of k scalar vectors (k = 1 but in a batch)
//
// With full tables (t = nwin, the default; the CRS is static and a 2^20-term G1
// table is ~1 GB) all windows feed ONE bucket set and the final result is a single
// sum_b b * S_b — no per-window reduction, no Horner doublings on the critical path.
// A reduced table (t < nwin rows) stores only 2^(c*j) * P_i for j < t: window w
// reads row j = w mod t and feeds the buckets of group g = w / t, and the tail
// returns sum_g 2^(c*t*g) * sum_b b * S_(g,b) (one Horner chain over all groups).
//
// Pipeline per MSM (one stream, no host sync):
//   k_digits_count   signed-digit recode, histogram of bucket sizes (RED.ADD)
//   k_scan           exclusive prefix sum -> bucket offsets
//   k_digits_scatter recode again, scatter entry ids into bucket order
//   k_accumulate     LPB lanes per bucket slice: gather + XYZZ mixed add, then a
//                    warp-shuffle tree merges the LPB partial sums
//   k_merge_slices   buckets that were cut into slices (skewed scalars) are re-joined
//   k_bucket_reduce  sum_b b*S_b by segments (running sums + small scalar mul)
//   k_sum_points     tree-sum of the segment results -> one XYZZ record
#pragma once
#include <cuda_runtime.h>

#include "ec.cuh"

namespace b200 {

// ------------------------------------------------------------ vector loads
// A 32 B-aligned field element as two 128-bit global loads (sm_90 has no 256-bit load; both halves hit the same
// 32-byte sector).
__device__ __forceinline__ void ld256(const void* p, uint32_t* o) {
  uint64_t a, b, c, d;
#ifdef __CUDA_ARCH__
  asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p));
  asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2+16];" : "=l"(c), "=l"(d) : "l"(p));
#else  // g++ test vehicle (csrc/host_stub)
  const uint64_t* q = static_cast<const uint64_t*>(p);
  a = q[0]; b = q[1]; c = q[2]; d = q[3];
#endif
  o[0] = (uint32_t)a; o[1] = (uint32_t)(a >> 32);
  o[2] = (uint32_t)b; o[3] = (uint32_t)(b >> 32);
  o[4] = (uint32_t)c; o[5] = (uint32_t)(c >> 32);
  o[6] = (uint32_t)d; o[7] = (uint32_t)(d >> 32);
}
// Same, for random gathers of 64-byte points: ask L2 to fetch only the 64 B it needs (LDG...LTC64B)
// rather than the whole 128-byte line.
__device__ __forceinline__ void ld256_g64(const void* p, uint32_t* o) {
  uint64_t a, b, c, d;
#ifdef __CUDA_ARCH__
  asm volatile("ld.global.nc.L2::64B.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p));
  asm volatile("ld.global.nc.L2::64B.v2.u64 {%0,%1}, [%2+16];" : "=l"(c), "=l"(d) : "l"(p));
#else
  const uint64_t* q = static_cast<const uint64_t*>(p);
  a = q[0]; b = q[1]; c = q[2]; d = q[3];
#endif
  o[0] = (uint32_t)a; o[1] = (uint32_t)(a >> 32);
  o[2] = (uint32_t)b; o[3] = (uint32_t)(b >> 32);
  o[4] = (uint32_t)c; o[5] = (uint32_t)(c >> 32);
  o[6] = (uint32_t)d; o[7] = (uint32_t)(d >> 32);
}
template <class P, bool I>
__device__ __forceinline__ Affine<Fp<P, I>> ld_affine_gather(const Affine<Fp<P, I>>* p) {
  Affine<Fp<P, I>> r;
  ld256_g64(&p->x, r.x.l);
  ld256_g64(&p->y, r.y.l);
  return r;
}
template <class P, bool I>
__device__ __forceinline__ Fp<P, I> ld_fe(const Fp<P, I>* p) { Fp<P, I> r; ld256(p, r.l); return r; }
template <bool I>
__device__ __forceinline__ Fq2T<I> ld_fe(const Fq2T<I>* p) { Fq2T<I> r; ld256(&p->c0, r.c0.l); ld256(&p->c1, r.c1.l); return r; }
template <class F>
__device__ __forceinline__ Affine<F> ld_affine(const Affine<F>* p) {
  Affine<F> r;
  r.x = ld_fe(&p->x);
  r.y = ld_fe(&p->y);
  return r;
}

template <bool I>
__device__ __forceinline__ Affine<Fq2T<I>> ld_affine_gather(const Affine<Fq2T<I>>* p) { return ld_affine(p); }  // 128 B = a full line

template <class T>
__device__ __forceinline__ T shfl_down_struct(const T& v, int delta, int width) {
  static_assert(sizeof(T) % 4 == 0, "");
  T r;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&v);
  uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int i = 0; i < (int)(sizeof(T) / 4); i++) d[i] = __shfl_down_sync(0xffffffffu, s[i], delta, width);
  return r;
}

// -------------------------------------------------------------- base upload
// Standard-form Jacobian -> Montgomery affine (table window 0).  err |= 1 when a
// coordinate is >= q.
template <class F>
__global__ void k_load_bases(const F* __restrict__ jac_std, size_t n, Affine<F>* __restrict__ out, int* err) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F X = jac_std[3 * i], Y = jac_std[3 * i + 1], Z = jac_std[3 * i + 2];
  if (X.geq_modulus() || Y.geq_modulus() || Z.geq_modulus()) {
    atomicOr(err, 1);
    out[i] = Affine<F>::inf();
    return;
  }
  Jacobian<F> p{X.to_mont(), Y.to_mont(), Z.to_mont()};
  Affine<F> a;
  if (p.Z == F::one())
    a = Affine<F>{p.X, p.Y};
  else
    a = jac_to_affine(p);
  out[i] = a;
}

// state[i] <- 2^c * state[i]   (XYZZ running point of the window precompute)
template <class F>
__global__ void k_window_step(XYZZ<F>* state, size_t n, int c) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  XYZZ<F> p = state[i];
  for (int k = 0; k < c; k++) p = xyzz_dbl(p);
  state[i] = p;
}
template <class F>
__global__ void k_affine_to_xyzz(const Affine<F>* in, XYZZ<F>* out, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = XYZZ<F>::from_affine(in[i]);
}
// Batch normalisation with Montgomery's trick, K points per thread: one field
// inversion per K points.
template <class F, int K>
__global__ void k_batch_to_affine(const XYZZ<F>* __restrict__ in, Affine<F>* __restrict__ out, size_t n) {
  size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t base = t * K;
  if (base >= n) return;
  F pre[K];  // prefix products of d_k = ZZ_k * ZZZ_k (skipping infinities)
  F acc = F::one();
  int cnt = (int)((n - base) < (size_t)K ? (n - base) : (size_t)K);
  for (int k = 0; k < cnt; k++) {
    pre[k] = acc;
    XYZZ<F> p = in[base + k];
    if (!p.is_inf()) acc = acc * (p.ZZ * p.ZZZ);
  }
  F inv = acc.inverse();
  for (int k = cnt - 1; k >= 0; k--) {
    XYZZ<F> p = in[base + k];
    if (p.is_inf()) {
      out[base + k] = Affine<F>::inf();
      continue;
    }
    F i = inv * pre[k];              // 1 / (ZZ*ZZZ)
    inv = inv * (p.ZZ * p.ZZZ);
    out[base + k] = Affine<F>{p.X * (i * p.ZZZ), p.Y * (i * p.ZZ)};
  }
}

// ------------------------------------------------------------ digit recode
struct MsmShape {
  uint32_t n;      // terms
  uint32_t c;      // window bits
  uint32_t nwin;   // ceil(255 / c)
  uint32_t nbuckets;  // 2^(c-1): buckets of one window group
  uint32_t table_stride;  // points per window in the table (>= n)
  uint32_t rows = nwin;   // table rows t: window w reads row w mod t (nwin = full tables)
  uint32_t groups = 1;    // ceil(nwin / rows) window groups, buckets g*nbuckets + 1 .. (g+1)*nbuckets
  // k scalar vectors over the same bases (b200_msm_device_batch): term i of vector p is scalar p*vec_stride + i times
  // base i, and vector p owns window groups p*groups .. (p+1)*groups - 1 of the bucket range
  uint32_t vecs = 1;
  uint32_t vec_stride = 0;
};

// Buckets over all window groups of all vectors: the range of the counting sort, the slice tables and the accumulation.
__host__ __device__ __forceinline__ uint32_t total_buckets(const MsmShape& sh) { return sh.vecs * sh.groups * sh.nbuckets; }

// Signed-digit windows of a 254-bit scalar: digit w in (-2^(c-1), 2^(c-1)].
// Calls f(w, bucket, sign) for every non-zero digit.
template <class Fn>
__device__ __forceinline__ void for_each_digit(const uint32_t* s, const MsmShape& sh, Fn&& f) {
  uint32_t carry = 0;
  const uint32_t half = 1u << (sh.c - 1);
  const uint32_t mask = (sh.c == 32) ? 0xffffffffu : ((1u << sh.c) - 1u);
  for (uint32_t w = 0; w < sh.nwin; w++) {
    uint32_t bit = w * sh.c;
    uint32_t idx = bit >> 5, sft = bit & 31;
    uint64_t lo = idx < 8 ? s[idx] : 0u;
    uint64_t hi = idx + 1 < 8 ? s[idx + 1] : 0u;
    uint32_t raw = (uint32_t)(((lo | (hi << 32)) >> sft) & mask) + carry;
    uint32_t neg = raw > half;
    uint32_t bucket = neg ? ((1u << sh.c) - raw) : raw;
    carry = neg;
    if (bucket) f(w, bucket, neg);
  }
}

__device__ __forceinline__ void load_scalar(const Fr* scalars, size_t i, int mont, uint32_t* s, int* err) {
  Fr v = ld_fe(&scalars[i]);
  if (mont) v = v.from_mont();
  else if (v.geq_modulus()) {
    atomicOr(err, 2);
    v = Fr::zero();
  }
#pragma unroll
  for (int k = 0; k < 8; k++) s[k] = v.l[k];
}

// Where the digit |d| of window w goes: table row w mod t, bucket id (vg + g)*2^(c-1) + |d| of group g = w / t, with vg
// the first group of the term's scalar vector.
__device__ __forceinline__ uint32_t digit_row(const MsmShape& sh, uint32_t w, uint32_t d, uint32_t& bucket_id, uint32_t vg = 0) {
  const uint32_t g = sh.groups > 1 ? w / sh.rows : 0u;
  bucket_id = (vg + g) * sh.nbuckets + d;
  return w - g * sh.rows;
}

// Thread i of the recode kernels takes term i of vector i / n (one vector: term i).  Returns false past the last term;
// `vg` is the vector's first window group and `si` the scalar's index.
__device__ __forceinline__ bool batch_term(const MsmShape& sh, size_t& i, size_t& si, uint32_t& vg) {
  if (sh.vecs == 1) {
    si = i;
    vg = 0;
    return i < sh.n;
  }
  const size_t p = i / sh.n;
  if (p >= sh.vecs) return false;
  i -= p * sh.n;
  si = p * sh.vec_stride + i;
  vg = (uint32_t)p * sh.groups;
  return true;
}

__global__ void k_digits_count(const Fr* __restrict__ scalars, MsmShape sh, int mont, uint32_t* counts, int* err) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, si;
  uint32_t vg;
  if (!batch_term(sh, i, si, vg)) return;
  uint32_t s[8];
  load_scalar(scalars, si, mont, s, err);
  for_each_digit(s, sh, [&](uint32_t w, uint32_t d, uint32_t) {
    uint32_t bucket;
    digit_row(sh, w, d, bucket, vg);
    atomicAdd(&counts[bucket], 1u);
  });
}

__global__ void k_digits_scatter(const Fr* __restrict__ scalars, MsmShape sh, int mont, uint32_t* cursor,
                                 uint32_t* __restrict__ entries, int* err) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, si;
  uint32_t vg;
  if (!batch_term(sh, i, si, vg)) return;
  uint32_t s[8];
  load_scalar(scalars, si, mont, s, err);
  for_each_digit(s, sh, [&](uint32_t w, uint32_t d, uint32_t neg) {
    uint32_t bucket;
    const uint32_t row = digit_row(sh, w, d, bucket, vg);
    uint32_t pos = atomicAdd(&cursor[bucket], 1u);
    entries[pos] = ((row * sh.table_stride + (uint32_t)i) << 1) | neg;
  });
}

// Exclusive scan of counts[0..m) -> offsets[0..m], cursor = copy of offsets, and
// the SLICE tables: a bucket holding more than `cap` entries is cut into
// ceil(cnt/cap) equal slices so that skewed scalar distributions (small witness
// values, a sparse top window, all-ones) cannot serialise on one bucket.  One
// block; thread t owns a contiguous run of buckets.
struct SliceTables {
  uint32_t* slice_off;     // [m+1] first slice id of each bucket (bucket 0 owns none)
  uint32_t* slice_start;   // [max_slices]
  uint32_t* slice_end;     // [max_slices]
};
// fixed != 0: slices hold exactly `cap` entry slots (last one of a bucket partially filled) — the
// perfect-binary-tree layout of the batched-affine accumulation.
//
// The counters of a batch of k scalar vectors (k*G*2^(c-1) of them) are scanned by several blocks: block b takes counters
// [b*chunk, (b+1)*chunk), k_scan_totals first writes every block's packed (entries, slices) total, and block b starts
// from the sum of the totals before it.  One block (chunk >= m, no totals) is the single-MSM scan.
__device__ __forceinline__ unsigned long long scan_item(const uint32_t* counts, uint32_t k, uint32_t hi, uint32_t cap) {
  uint32_t c = k < hi ? counts[k] : 0u;
  uint32_t sl = (k == 0 || k >= hi) ? 0u : (c <= cap ? 1u : (c + cap - 1) / cap);
  return ((unsigned long long)sl << 32) | c;
}
__global__ void __launch_bounds__(1024) k_scan_totals(const uint32_t* __restrict__ counts, uint32_t m, uint32_t cap,
                                                      uint32_t chunk, unsigned long long* __restrict__ totals) {
  __shared__ unsigned long long tot_s;
  const uint32_t lo = blockIdx.x * chunk, hi = m - lo < chunk ? m : lo + chunk;
  if (threadIdx.x == 0) tot_s = 0ull;
  __syncthreads();
  unsigned long long v = 0ull;
  for (uint32_t k = lo + threadIdx.x; k < hi; k += blockDim.x) v += scan_item(counts, k, hi, cap);
  if (v) atomicAdd(&tot_s, v);
  __syncthreads();
  if (threadIdx.x == 0) totals[blockIdx.x] = tot_s;
}
__global__ void __launch_bounds__(1024) k_scan(const uint32_t* __restrict__ counts, uint32_t m, uint32_t cap, int fixed,
                                               uint32_t* offsets, uint32_t* cursor, SliceTables st,
                                               uint32_t chunk = 0xffffffffu, const unsigned long long* totals = nullptr) {
  // One block walks its counters in coalesced tiles of blockDim.x; (entry count, slice count) are packed into one
  // 64-bit value so a single warp-shuffle scan + a scan of the warp totals serves both prefix sums.  (The first version
  // gave every thread 64 consecutive counters: uncoalesced and serial.)
  __shared__ unsigned long long wsum[32];
  __shared__ unsigned long long carry_s;
  const uint32_t t = threadIdx.x, T = blockDim.x, lane = t & 31u, warp = t >> 5, nwarps = T >> 5;
  const uint32_t lo = blockIdx.x * chunk, hi = m - lo < chunk ? m : lo + chunk;
  if (t == 0) carry_s = 0ull;
  __syncthreads();
  if (totals) {   // the blocks before this one
    unsigned long long before = 0ull;
    for (uint32_t j = t; j < blockIdx.x; j += T) before += totals[j];
    if (before) atomicAdd(&carry_s, before);
    __syncthreads();
  }
  for (uint32_t base = lo; base < hi; base += T) {
    uint32_t k = base + t;
    unsigned long long v = scan_item(counts, k, hi, cap), incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      unsigned long long up = __shfl_up_sync(0xffffffffu, incl, off);
      if ((int)lane >= off) incl += up;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      unsigned long long w = lane < nwarps ? wsum[lane] : 0ull, wi = w;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        unsigned long long up = __shfl_up_sync(0xffffffffu, wi, off);
        if ((int)lane >= off) wi += up;
      }
      wsum[lane] = wi - w;   // exclusive prefix of the warp totals; lane 31's inclusive value is the tile total
    }
    __syncthreads();
    unsigned long long carry = carry_s;
    unsigned long long excl = carry + wsum[warp] + (incl - v);
    if (k < hi) {
      uint32_t run = (uint32_t)excl, srun = (uint32_t)(excl >> 32);
      offsets[k] = run;
      cursor[k] = run;
      st.slice_off[k] = srun;
    }
    __syncthreads();
    if (t == T - 1) carry_s = excl + v;   // inclusive prefix of the tile's last element = new carry
    __syncthreads();
  }
  if (t == 0 && hi == m) {
    unsigned long long tot = carry_s;
    offsets[m] = (uint32_t)tot;
    st.slice_off[m] = (uint32_t)(tot >> 32);
  }
  (void)fixed;
}

// slice_start / slice_end of every slice, one thread per bucket (k_scan wrote slice_off and offsets)
__global__ void k_fill_slices(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ offsets, uint32_t m,
                              uint32_t cap, int fixed, SliceTables st) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x + 1;
  if (k >= m) return;
  uint32_t c = counts[k], run = offsets[k], s0 = st.slice_off[k];
  uint32_t ns = c <= cap ? 1 : (c + cap - 1) / cap;
  uint32_t each = fixed ? cap : (c + ns - 1) / ns;
  for (uint32_t j = 0; j < ns; j++) {
    uint32_t b0 = run + j * each, b1 = b0 + each;
    st.slice_start[s0 + j] = b0 < run + c ? b0 : run + c;
    st.slice_end[s0 + j] = b1 < run + c ? b1 : run + c;
  }
}

// ------------------------------------------------------- bucket accumulate
// LPB lanes cooperate on one slice (normally = one bucket): lane l takes entries
// l, l+LPB, ... (coalesced reads of `entries`), gathers the precomputed affine
// points and mixed-adds them; a warp-shuffle tree then merges the LPB partials.
// (A software-prefetch variant — next point fetched before the current add — and 80..154-register builds were
// no faster: the kernel is bound by the multiply pipe.)
template <class F, int LPB, int MINB = 1>
__global__ void __launch_bounds__(128, MINB)
k_accumulate(const Affine<F>* __restrict__ table, const uint32_t* __restrict__ entries, SliceTables st,
             uint32_t m, XYZZ<F>* __restrict__ slice_out) {
  uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t sid = gt / LPB;
  uint32_t lane = gt % LPB;
  uint32_t nslices = st.slice_off[m];
  bool live = sid < nslices;
  uint32_t start = live ? st.slice_start[sid] : 0, end = live ? st.slice_end[sid] : 0;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint32_t k = start + lane; k < end; k += LPB) {
    uint32_t e = entries[k];
    Affine<F> p = ld_affine_gather(&table[e >> 1]);
    if (e & 1) p.y = p.y.neg();
    xyzz_madd(acc, p);
  }
#pragma unroll
  for (int off = LPB / 2; off > 0; off >>= 1) {
    XYZZ<F> other = shfl_down_struct(acc, off, LPB);
    xyzz_add(acc, other);
  }
  if (live && lane == 0) slice_out[sid] = acc;
}

// buckets[b-1] = sum of the slices of bucket b.  Thread per bucket copies the
// common single-slice case; buckets that were split are then summed by the whole
// warp, one after another.
template <class F>
__global__ void __launch_bounds__(128)
k_merge_slices(const XYZZ<F>* __restrict__ slice_out, SliceTables st, uint32_t nbuckets,
               XYZZ<F>* __restrict__ buckets) {
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x + 1;
  uint32_t lane = threadIdx.x & 31;
  uint32_t first = 0, cnt = 0;
  if (b <= nbuckets) {
    first = st.slice_off[b];
    cnt = st.slice_off[b + 1] - first;
    if (cnt == 1) buckets[b - 1] = slice_out[first];
  }
  uint32_t multi = __ballot_sync(0xffffffffu, cnt > 1);
  while (multi) {
    int j = __ffs(multi) - 1;
    multi &= multi - 1;
    uint32_t f = __shfl_sync(0xffffffffu, first, j), c = __shfl_sync(0xffffffffu, cnt, j);
    uint32_t bj = __shfl_sync(0xffffffffu, b, j);
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t k = lane; k < c; k += 32) xyzz_add(acc, slice_out[f + k]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      XYZZ<F> other = shfl_down_struct(acc, off, 32);
      xyzz_add(acc, other);
    }
    if (lane == 0) buckets[bj - 1] = acc;
  }
}

// acc <- m * acc for a small integer m (MSB-first double-and-add)
template <class F>
__device__ __forceinline__ XYZZ<F> xyzz_mul_small(const XYZZ<F>& p, uint32_t m) {
  XYZZ<F> r = XYZZ<F>::inf();
  for (int bit = 31 - __clz(m | 1); bit >= 0; bit--) {
    r = xyzz_dbl(r);
    if ((m >> bit) & 1) xyzz_add(r, p);
  }
  return m ? r : XYZZ<F>::inf();
}

// Segment t covers buckets [t*seg+1, (t+1)*seg]: out[t] = sum_b b * S_b over the segment.  Window group y = blockIdx.y
// reads its own nbuckets buckets, writes its own nseg records and scales them by 2^(g*gshift) (gshift = c*t): g = y for
// one MSM, g = y mod `groups` in a batch of scalar vectors (BATCH, a separate instantiation: the one-MSM kernel is unchanged).
template <class F, bool BATCH = false>
__global__ void __launch_bounds__(128)
k_bucket_reduce(const XYZZ<F>* __restrict__ buckets, uint32_t nbuckets, uint32_t seg, XYZZ<F>* __restrict__ out,
                uint32_t nseg, uint32_t gshift = 0, uint32_t groups = 1) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nseg) return;
  const uint32_t y = blockIdx.y, g = BATCH ? y % groups : y;
  buckets += (size_t)y * nbuckets;
  out += (size_t)y * nseg;
  uint32_t lo = t * seg + 1;
  uint32_t hi = lo + seg - 1 < nbuckets ? lo + seg - 1 : nbuckets;
  XYZZ<F> acc = XYZZ<F>::inf(), sum = XYZZ<F>::inf();
  for (uint32_t b = hi; b >= lo; b--) {
    xyzz_add(acc, buckets[b - 1]);
    xyzz_add(sum, acc);
  }
  XYZZ<F> scaled = xyzz_mul_small(acc, lo - 1);
  xyzz_add(sum, scaled);
  for (uint32_t k = 0; k < g * gshift; k++) sum = xyzz_dbl(sum);
  out[t] = sum;
}

// out[blockIdx.x] = sum of this block's contiguous chunk of `per_block` inputs (strided accumulate, warp
// shuffle tree, then warp 0 folds the 8 warp sums with a second shuffle tree).  Launched with one block it is
// the final tree sum; with several blocks it is the first level of a two-level sum (shorter latency chain).
template <class F>
__global__ void __launch_bounds__(256)
k_sum_points(const XYZZ<F>* __restrict__ in, uint32_t count, uint32_t per_block, XYZZ<F>* __restrict__ out) {
  __shared__ XYZZ<F> warp_sums[8];
  uint32_t t = threadIdx.x;
  uint32_t lo = blockIdx.x * per_block;
  uint32_t hi = lo + per_block < count ? lo + per_block : count;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint32_t k = lo + t; k < hi; k += blockDim.x) xyzz_add(acc, in[k]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    XYZZ<F> other = shfl_down_struct(acc, off, 32);
    xyzz_add(acc, other);
  }
  if ((t & 31) == 0) warp_sums[t >> 5] = acc;
  __syncthreads();
  if (t < 32) {
    XYZZ<F> r = t < (blockDim.x >> 5) ? warp_sums[t] : XYZZ<F>::inf();
#pragma unroll
    for (int off = 4; off > 0; off >>= 1) {
      XYZZ<F> other = shfl_down_struct(r, off, 8);
      xyzz_add(r, other);
    }
    if (t == 0) out[blockIdx.x] = r;
  }
}

// ---- weighted bucket reduction with a short dependency chain ---------------------------------------------------------
// sum_{b=1..B} b * S_b (buckets[b-1] = S_b, B = 2^(c-1)) without running sums: with b - 1 = hi*K + lo (K = 2^kl),
//     sum b S_b = K * sum_hi hi * R_hi + sum_lo lo * C_lo + sum_hi R_hi,   R_hi = sum_lo S_(hi,lo),  C_lo = sum_hi S_(hi,lo)
// (1) k_tail_rowcol: one warp per row and per column (strided adds + a 5-level shuffle tree);
// (2) k_tail_planes: sum_i i * P_i over <= K points by bit planes, one warp per (group, bit): T_j = sum over the i with
//     bit j set, plus one warp for the plain sum of the rows;
// (3) k_tail_horner: the c-1 planes of the combined weight (low kl bits from the columns, high bits from the rows) in one
//     Horner chain of c-1 doublings and additions, plus the plain sum.
// Depth: ~(K/32 + 5) + (K/32 + 5) + 2(c-1) dependent group operations instead of 2*seg + 16 doublings + ... per thread
// followed by two more tree levels, on the serial tail of every MSM
// (stand-alone MSM latency, and the per-rank critical path when a proof is sharded over 8 GPUs).
template <class F>
__device__ __forceinline__ XYZZ<F> warp_sum_xyzz(XYZZ<F> acc) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    XYZZ<F> other = shfl_down_struct(acc, off, 32);
    xyzz_add(acc, other);
  }
  return acc;   // lane 0 holds the sum
}
// warps [0, H): R[hi];  warps [H, H+K): C[lo]      (H = B / K rows of K buckets)
// Window group g = blockIdx.y reads buckets [g*B, (g+1)*B) and writes R[g*H ..], C[g*K ..].
template <class F>
__global__ void __launch_bounds__(128) k_tail_rowcol(const XYZZ<F>* __restrict__ buckets, uint32_t kl, uint32_t H,
                                                     XYZZ<F>* __restrict__ R, XYZZ<F>* __restrict__ C) {
  const uint32_t K = 1u << kl;
  uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (w >= H + K) return;
  const uint32_t g = blockIdx.y;
  buckets += ((size_t)g * H) << kl;
  R += (size_t)g * H;
  C += (size_t)g * K;
  XYZZ<F> acc = XYZZ<F>::inf();
  if (w < H) {
    for (uint32_t lo = lane; lo < K; lo += 32) xyzz_add(acc, buckets[((size_t)w << kl) + lo]);
  } else {
    uint32_t lo = w - H;
    for (uint32_t hi = lane; hi < H; hi += 32) xyzz_add(acc, buckets[((size_t)hi << kl) + lo]);
  }
  acc = warp_sum_xyzz(acc);
  if (lane == 0) (w < H ? R[w] : C[w - H]) = acc;
}
// planes[j] for j < kl: sum of C[i] over i with bit j set; planes[kl + j] for j < kh: sum of R[i] over i with bit j set;
// planes[kl + kh]: sum of all R[i].   One warp per plane; window group g = blockIdx.y has its own R, C and kl + kh + 1 planes.
template <class F>
__global__ void __launch_bounds__(128) k_tail_planes(const XYZZ<F>* __restrict__ R, const XYZZ<F>* __restrict__ C, uint32_t kl,
                                                     uint32_t kh, XYZZ<F>* __restrict__ planes) {
  uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (w > kl + kh) return;
  const uint32_t g = blockIdx.y;
  R += (size_t)g << kh;
  C += (size_t)g << kl;
  planes += (size_t)g * (kl + kh + 1);
  const XYZZ<F>* src = w < kl ? C : R;
  const uint32_t n = w < kl ? (1u << kl) : (1u << kh);
  const uint32_t bit = w < kl ? w : w - kl;
  const bool all = w == kl + kh;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint32_t i = lane; i < n; i += 32)
    if (all || ((i >> bit) & 1u)) xyzz_add(acc, src[i]);
  acc = warp_sum_xyzz(acc);
  if (lane == 0) planes[w] = acc;
}
// Row chunks of the tail kernels that take (vector, window group) as blockIdx.y: launch(y0, ny) for consecutive chunks of
// the vecs*groups rows, each at most max_rows rows (65535 on the device: the gridDim.y limit) and a multiple of groups,
// so that blockIdx.y mod groups inside a chunk is still the window group.
template <class Fn>
inline void for_each_tail_chunk(const MsmShape& sh, uint32_t max_rows, Fn&& launch) {
  const uint32_t rows = sh.vecs * sh.groups, whole = max_rows / sh.groups, chunk = (whole ? whole : 1u) * sh.groups;
  for (uint32_t y0 = 0; y0 < rows; y0 += chunk) launch(y0, rows - y0 < chunk ? rows - y0 : chunk);
}

// out = sum_g 2^(g*gshift) (sum_{j < nplanes} 2^j P_g[j] + P_g[nplanes]) over `groups` window groups, P_g = planes +
// g*(nplanes + 1) and gshift = c*t (one group: the full-table tail).  The bit positions p = g*gshift + j, 0 <= p < npos,
// form one Horner chain; positions nplanes <= j < gshift of a group hold no plane.  One warp; lane q < 16 takes `per`
// consecutive positions, shifts its partial sum by q * per doublings, and a 4-level shuffle tree adds the 16 partial sums:
// ~npos + 5 dependent group operations (npos ~ 255 for a reduced table) instead of 2 * npos for a single Horner chain.
// Block v runs the chain of scalar vector v of a batch: its groups * (nplanes + 1) planes, record out[v].
template <class F>
__global__ void __launch_bounds__(32) k_tail_horner(const XYZZ<F>* __restrict__ planes, uint32_t nplanes, XYZZ<F>* __restrict__ out,
                                                    uint32_t groups = 1, uint32_t gshift = 0) {
  planes += (size_t)blockIdx.x * groups * (nplanes + 1);
  out += blockIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t npos = (groups - 1) * gshift + nplanes;
  const uint32_t per = (npos + 15) / 16;
  XYZZ<F> acc = XYZZ<F>::inf();
  if (lane < 16) {
    const uint32_t lo = lane * per, hi = lo + per < npos ? lo + per : npos;
    for (int p = (int)hi - 1; p >= (int)lo; p--) {
      acc = xyzz_dbl(acc);
      const uint32_t g = groups > 1 ? (uint32_t)p / gshift : 0u, j = (uint32_t)p - g * gshift;
      const XYZZ<F>* pg = planes + (size_t)g * (nplanes + 1);
      if (j < nplanes) xyzz_add(acc, pg[j]);
      if (j == 0 && g > 0) xyzz_add(acc, pg[nplanes]);   // plain sum of group g, weight 2^(g*gshift)
    }
    if (lo < npos)
      for (uint32_t d = 0; d < lo; d++) acc = xyzz_dbl(acc);
    if (lane == 0) xyzz_add(acc, planes[nplanes]);
  }
#pragma unroll
  for (int off = 8; off > 0; off >>= 1) {
    XYZZ<F> other = shfl_down_struct(acc, off, 32);
    xyzz_add(acc, other);
  }
  if (lane == 0) out[0] = acc;
}

// XYZZ (Montgomery) -> standard-form Jacobian (x, y, 1), infinity -> zeros.
template <class F>
__global__ void k_finalize(const XYZZ<F>* in, F* out_jac_std) {
  if (threadIdx.x | blockIdx.x) return;
  Affine<F> a = xyzz_to_affine<F, true>(in[0]);
  if (a.is_inf()) {
    out_jac_std[0] = F::zero();
    out_jac_std[1] = F::zero();
    out_jac_std[2] = F::zero();
  } else {
    out_jac_std[0] = a.x.from_mont();
    out_jac_std[1] = a.y.from_mont();
    F one = F::zero();
    reinterpret_cast<uint32_t*>(&one)[0] = 1;
    out_jac_std[2] = one;
  }
}

// --------------------------------------- reference-order batch scalar mul
// One thread per term: bn128/g1.go:140-155 (MSB-first over BitLen bits, q starts
// at (0,0,0)) with the reference's own add/double formulas => X,Y,Z-exact.
template <class F>
__global__ void __launch_bounds__(128)
k_mul_batch_ref(const F* __restrict__ pts_jac_std, int bcast, const Fr* __restrict__ scalars, size_t n,
                F* __restrict__ out_jac_std, int* err) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  size_t pi = bcast ? 0 : i;
  F X = pts_jac_std[3 * pi], Y = pts_jac_std[3 * pi + 1], Z = pts_jac_std[3 * pi + 2];
  if (X.geq_modulus() || Y.geq_modulus() || Z.geq_modulus()) atomicOr(err, 1);
  Jacobian<F> p{X.to_mont(), Y.to_mont(), Z.to_mont()};
  Fr s = scalars[i];
  Jacobian<F> q = Jacobian<F>::inf();
  bool started = false;
  for (int w = 7; w >= 0; w--) {
    uint32_t limb = s.l[w];
    for (int b = 31; b >= 0; b--) {
      uint32_t bit = (limb >> b) & 1;
      if (!started && !bit) continue;  // BitLen() skips leading zeros
      started = true;
      q = jac_double_ref(q);
      if (bit) q = jac_add_ref(q, p);
    }
  }
  out_jac_std[3 * i] = q.X.from_mont();
  out_jac_std[3 * i + 1] = q.Y.from_mont();
  out_jac_std[3 * i + 2] = q.Z.from_mont();
}

}  // namespace b200
