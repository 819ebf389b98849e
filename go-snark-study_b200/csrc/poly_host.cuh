// Host-side orchestration of the F_r polynomial kernels (ntt.cuh): transform
// plans, multiplication, power-series inversion and division with a cached
// transformed inverse for a fixed divisor (pk.Z).  Included by capi.cu only.
#pragma once
#include <map>
#include <memory>

#include "ntt.cuh"

// Kernel launches of the polynomial orchestration go through these two macros so that the SAME host code (transform
// plans, division, interpolation, subproduct trees) also runs in the CPU test vehicle (tests/host: the macros become
// loops over emulated CTAs).  _CTA marks kernels that synchronise inside a block.
#ifndef B200_LAUNCH
#define B200_LAUNCH(kernel, grid, block, stream, ...) kernel<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__)
#define B200_LAUNCH_CTA(kernel, grid, block, stream, ...) kernel<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__)
#endif

namespace b200 {

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t b) {
    if (p) cudaFree(p);
    p = nullptr;
    bytes = b;
    return b ? cudaMalloc(&p, b) : cudaSuccess;
  }
  cudaError_t ensure(size_t b) { return b <= bytes && p ? cudaSuccess : alloc(b); }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

inline unsigned nblk(size_t n, unsigned bs) { return (unsigned)((n + bs - 1) / bs); }
inline int ceil_log2(size_t n) {
  int k = 0;
  while (((size_t)1 << k) < n) k++;
  return k;
}

// host-side F_r helpers (the arithmetic headers compile for the host too)
inline Fr fr_from_u64(uint64_t v) {
  Fr r = Fr::zero();
  r.l[0] = (uint32_t)v;
  r.l[1] = (uint32_t)(v >> 32);
  return r.to_mont();
}
inline Fr fr_pow2k(Fr b, int k) {  // b^(2^k)
  for (int i = 0; i < k; i++) b = b.sqr();
  return b;
}

struct NttPlan {
  int logn = 0;
  DevBuf tw, tw_inv;  // N/2 powers of w and of w^-1
  Fr n_inv;           // N^-1 (Montgomery)
};

struct PolyCtx {
  // Transforms of >= 2^10 points run as fused shared-memory passes (ntt.cuh: k_ntt_fused; 3 passes instead of 21 stage
  // launches at 2^21 points); bit-identical to the stage kernels.
  static constexpr bool fused() { return true; }
  unsigned long long* launch_counter = nullptr;
  void note(unsigned n) { if (launch_counter) *launch_counter += n; }
  std::map<int, std::unique_ptr<NttPlan>> plans;
  DevBuf bufA, bufB, bufC;  // transform workspaces

  cudaError_t plan(int logn, NttPlan** out, cudaStream_t st) {
    auto it = plans.find(logn);
    if (it != plans.end()) {
      *out = it->second.get();
      return cudaSuccess;
    }
    auto p = std::make_unique<NttPlan>();
    p->logn = logn;
    size_t N = (size_t)1 << logn;
    Fr root;
    for (int i = 0; i < 8; i++) root.l[i] = FrParams::ROOT(i);
    Fr w = fr_pow2k(root, FrParams::TWO_ADICITY - logn);  // primitive N-th root of unity
    Fr w_inv = w.inverse_impl();
    p->n_inv = fr_from_u64(N).inverse_impl();
    size_t half = N / 2 ? N / 2 : 1;
    cudaError_t e;
    if ((e = p->tw.alloc(half * sizeof(Fr))) != cudaSuccess) return e;
    if ((e = p->tw_inv.alloc(half * sizeof(Fr))) != cudaSuccess) return e;
    B200_LAUNCH(k_twiddles, nblk(half, 256), 256, st, p->tw.as<Fr>(), (uint32_t)half, w);
    B200_LAUNCH(k_twiddles, nblk(half, 256), 256, st, p->tw_inv.as<Fr>(), (uint32_t)half, w_inv);
    *out = p.get();
    plans[logn] = std::move(p);
    return cudaGetLastError();
  }

  // natural -> bit-reversed
  cudaError_t forward(Fr* d, int logn, cudaStream_t st) {
    NttPlan* pl;
    cudaError_t e = plan(logn, &pl, st);
    if (e != cudaSuccess) return e;
    uint32_t N = 1u << logn, n_half = N >> 1;
    if (fused() && logn >= 10) {  // experiment: several stages per pass in shared memory (ntt.cuh: k_ntt_fused)
      unsigned passes = 0;
      ntt_fused_passes(logn, 0, [&](uint32_t log_hbot, uint32_t k) {
        B200_LAUNCH_CTA(k_ntt_fused, N / kNttTile, 256, st, d, pl->tw.as<Fr>(), n_half, log_hbot, k, 0);
        passes++;
      });
      note(passes);
      return cudaGetLastError();
    }
    for (uint32_t half = n_half; half >= 1; half >>= 1)
      B200_LAUNCH(k_ntt_dif_stage, nblk(n_half, 256), 256, st, d, pl->tw.as<Fr>(), n_half, half, n_half / half);
    note(logn);
    return cudaGetLastError();
  }
  // bit-reversed -> natural, WITHOUT the 1/N scale (callers fold it into a pointwise product)
  cudaError_t inverse_unscaled(Fr* d, int logn, cudaStream_t st) {
    NttPlan* pl;
    cudaError_t e = plan(logn, &pl, st);
    if (e != cudaSuccess) return e;
    uint32_t N = 1u << logn, n_half = N >> 1;
    if (fused() && logn >= 10) {
      unsigned passes = 0;
      ntt_fused_passes(logn, 1, [&](uint32_t log_hbot, uint32_t k) {
        B200_LAUNCH_CTA(k_ntt_fused, N / kNttTile, 256, st, d, pl->tw_inv.as<Fr>(), n_half, log_hbot, k, 1);
        passes++;
      });
      note(passes);
      return cudaGetLastError();
    }
    for (uint32_t half = 1; half <= n_half; half <<= 1)
      B200_LAUNCH(k_ntt_dit_stage, nblk(n_half, 256), 256, st, d, pl->tw_inv.as<Fr>(), n_half, half, n_half / half);
    note(logn);
    return cudaGetLastError();
  }
  // a <- a * b (both already forward-transformed, size N), scaled by 1/N so that
  // inverse_unscaled(a) yields the product coefficients.
  cudaError_t pointwise(Fr* a, const Fr* b, int logn, bool scale, cudaStream_t st) {
    NttPlan* pl;
    cudaError_t e = plan(logn, &pl, st);
    if (e != cudaSuccess) return e;
    uint32_t N = 1u << logn;
    B200_LAUNCH(k_pointwise_mul, nblk(N, 256), 256, st, a, b, N, pl->n_inv, scale ? 1 : 0);
    note(1);
    return cudaGetLastError();
  }
};

// A fixed divisor b (e.g. pk.Z): Montgomery copy + cached transformed inverse series.
struct Divisor {
  size_t nb = 0;
  DevBuf b_mont;      // nb coefficients, Montgomery, natural order
  // cache for one quotient length (a prove path always uses the same one)
  size_t nq = 0;
  int logn = 0;       // transform size of the quotient product
  DevBuf inv_ntt;     // forward transform of rev(b)^-1 mod x^nq, pre-scaled by 1/N
};

#define PCU(call)                          \
  do {                                     \
    cudaError_t e_ = (call);               \
    if (e_ != cudaSuccess) return e_;      \
  } while (0)

// g <- (rev(b))^-1 mod x^nq, Montgomery, written to out[0..nq)
inline cudaError_t series_inverse_rev(PolyCtx& pc, const Divisor& dv, size_t nq, Fr* out, int* d_err, cudaStream_t st) {
  int lp = ceil_log2(nq);
  size_t Pmax = (size_t)1 << lp;
  PCU(pc.bufA.ensure(4 * Pmax * sizeof(Fr)));
  PCU(pc.bufB.ensure(4 * Pmax * sizeof(Fr)));
  PCU(pc.bufC.ensure(2 * Pmax * sizeof(Fr)));
  Fr* A = pc.bufA.as<Fr>();
  Fr* B = pc.bufB.as<Fr>();
  Fr* g = pc.bufC.as<Fr>();  // current approximation, natural order
  const Fr* b = dv.b_mont.as<Fr>();
  uint32_t nb = (uint32_t)dv.nb;
  // f = rev(b): f[i] = b[nb-1-i]
  B200_LAUNCH(k_poly_load, 1, 32, st, b, nb, 1, 1, 1, A, 1, d_err);
  B200_LAUNCH(k_series_inv0, 1, 32, st, A, g, d_err);
  for (size_t P = 1; P < nq; P <<= 1) {
    int l4 = ceil_log2(4 * P);
    uint32_t N4 = 1u << l4;
    uint32_t take = (uint32_t)(2 * P < nb ? 2 * P : nb);
    B200_LAUNCH(k_poly_load, nblk(N4, 256), 256, st, b, nb, take, 1, 1, A, N4, d_err);            // f mod x^2P
    B200_LAUNCH(k_poly_load, nblk(N4, 256), 256, st, g, (uint32_t)P, (uint32_t)P, 0, 1, B, N4, d_err);  // g
    PCU(pc.forward(A, l4, st));
    PCU(pc.forward(B, l4, st));
    PCU(pc.pointwise(A, B, l4, true, st));
    PCU(pc.inverse_unscaled(A, l4, st));                     // A = f*g
    B200_LAUNCH(k_two_minus, nblk(N4, 256), 256, st, A, (uint32_t)(2 * P), N4);  // A = 2 - f*g mod x^2P
    PCU(pc.forward(A, l4, st));
    PCU(pc.pointwise(A, B, l4, true, st));
    PCU(pc.inverse_unscaled(A, l4, st));                     // A = g*(2 - f*g)
    PCU(cudaMemcpyAsync(g, A, 2 * P * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
  }
  PCU(cudaMemcpyAsync(out, g, nq * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
  return cudaGetLastError();
}

// Make sure dv caches the transformed inverse for quotient length nq.
inline cudaError_t divisor_prepare(PolyCtx& pc, Divisor& dv, size_t nq, int* d_err, cudaStream_t st) {
  if (dv.nq == nq && dv.inv_ntt.p) return cudaSuccess;
  int logn = ceil_log2(2 * nq - 1 > 1 ? 2 * nq - 1 : 2);
  size_t N = (size_t)1 << logn;
  PCU(dv.inv_ntt.alloc(N * sizeof(Fr)));
  Fr* inv = dv.inv_ntt.as<Fr>();
  PCU(cudaMemsetAsync(inv, 0, N * sizeof(Fr), st));
  PCU(series_inverse_rev(pc, dv, nq, inv, d_err, st));
  PCU(pc.forward(inv, logn, st));
  NttPlan* pl;
  PCU(pc.plan(logn, &pl, st));
  // fold the 1/N of the inverse transform into the cached operand
  B200_LAUNCH(k_scale, nblk(N, 256), 256, st, inv, (uint32_t)N, pl->n_inv);
  dv.nq = nq;
  dv.logn = logn;
  return cudaGetLastError();
}

// q = a div b (and optionally rem = a mod b), device buffers.
//   d_a      : na coefficients (standard form unless a_mont)
//   d_q_std  : nq = na - nb + 1 coefficients out, standard form, natural order
//   d_rem_std: nb - 1 coefficients out (standard form) or nullptr
inline cudaError_t poly_div_device(PolyCtx& pc, Divisor& dv, const Fr* d_a, size_t na, int a_mont, Fr* d_q_std,
                                   Fr* d_rem_std, int* d_err, cudaStream_t st) {
  size_t nb = dv.nb;
  size_t nq = na - nb + 1;
  PCU(divisor_prepare(pc, dv, nq, d_err, st));
  int logn = dv.logn;
  size_t N = (size_t)1 << logn;
  PCU(pc.bufA.ensure(N * sizeof(Fr)));
  Fr* X = pc.bufA.as<Fr>();
  // rev(a) mod x^nq, zero padded to N
  B200_LAUNCH(k_poly_load, nblk(N, 256), 256, st, d_a, (uint32_t)na, (uint32_t)nq, 1, a_mont, X, (uint32_t)N, d_err);
  PCU(pc.forward(X, logn, st));
  PCU(pc.pointwise(X, dv.inv_ntt.as<Fr>(), logn, false, st));  // 1/N already folded into inv_ntt
  PCU(pc.inverse_unscaled(X, logn, st));
  // rev(q) = X[0..nq)  ->  q natural order, standard form
  B200_LAUNCH(k_poly_store, nblk(nq, 256), 256, st, X, (uint32_t)nq, 1, 1, d_q_std);
  pc.note(2);
  if (d_rem_std && nb > 1) {
    int lr = ceil_log2(na);
    size_t Nr = (size_t)1 << lr;
    PCU(pc.bufA.ensure(Nr * sizeof(Fr)));
    PCU(pc.bufB.ensure(Nr * sizeof(Fr)));
    PCU(pc.bufC.ensure(Nr * sizeof(Fr)));
    Fr* Q = pc.bufA.as<Fr>();
    Fr* Bt = pc.bufB.as<Fr>();
    Fr* Am = pc.bufC.as<Fr>();
    B200_LAUNCH(k_poly_load, nblk(Nr, 256), 256, st, d_q_std, (uint32_t)nq, (uint32_t)nq, 0, 0, Q, (uint32_t)Nr, d_err);
    B200_LAUNCH(k_poly_load, nblk(Nr, 256), 256, st, dv.b_mont.as<Fr>(), (uint32_t)nb, (uint32_t)nb, 0, 1, Bt, (uint32_t)Nr, d_err);
    B200_LAUNCH(k_poly_load, nblk(Nr, 256), 256, st, d_a, (uint32_t)na, (uint32_t)na, 0, a_mont, Am, (uint32_t)Nr, d_err);
    PCU(pc.forward(Q, lr, st));
    PCU(pc.forward(Bt, lr, st));
    PCU(pc.pointwise(Q, Bt, lr, true, st));
    PCU(pc.inverse_unscaled(Q, lr, st));
    B200_LAUNCH(k_poly_sub_store, nblk(nb - 1, 256), 256, st, Am, Q, (uint32_t)(nb - 1), d_rem_std);
  }
  return cudaGetLastError();
}

// out = a * b (device, standard form in unless *_mont, standard form out), la + lb - 1 coefficients
inline cudaError_t poly_mul_device(PolyCtx& pc, const Fr* d_a, size_t la, int a_mont, const Fr* d_b, size_t lb,
                                   int b_mont, Fr* d_out_std, int* d_err, cudaStream_t st) {
  size_t lo = la + lb - 1;
  int logn = ceil_log2(lo > 1 ? lo : 2);
  size_t N = (size_t)1 << logn;
  PCU(pc.bufA.ensure(N * sizeof(Fr)));
  PCU(pc.bufB.ensure(N * sizeof(Fr)));
  Fr* A = pc.bufA.as<Fr>();
  Fr* B = pc.bufB.as<Fr>();
  B200_LAUNCH(k_poly_load, nblk(N, 256), 256, st, d_a, (uint32_t)la, (uint32_t)la, 0, a_mont, A, (uint32_t)N, d_err);
  B200_LAUNCH(k_poly_load, nblk(N, 256), 256, st, d_b, (uint32_t)lb, (uint32_t)lb, 0, b_mont, B, (uint32_t)N, d_err);
  PCU(pc.forward(A, logn, st));
  PCU(pc.forward(B, logn, st));
  PCU(pc.pointwise(A, B, logn, true, st));
  PCU(pc.inverse_unscaled(A, logn, st));
  B200_LAUNCH(k_poly_store, nblk(lo, 256), 256, st, A, (uint32_t)lo, 0, 1, d_out_std);
  return cudaGetLastError();
}

}  // namespace b200
