// Sparse QAP front end: witness + sparse R1CS -> ax, bx, cx, px at sizes where the reference's dense
// R1CSToQAP / CombinePolynomials (r1csqap/r1csqap.go:161-210) cannot be represented (m x n coefficients per
// matrix = 137 GB at n = 2^16, SURVEY H4).  Mathematically it IS CombinePolynomials(w, R1CSToQAP(a, b, c)):
//
//     ax = sum_i w_i * alpha_i(x),   alpha_i = LagrangeInterpolation of column i of A over x = 1..n   (:150-188)
//  => ax is the unique polynomial of degree < n with ax(j+1) = (A w)_j,   j = 0..n-1,
//
// so the three polynomials are obtained by one sparse mat-vec each and one interpolation over the
// arithmetic progression {1..n} each; px = ax*bx - cx (:204-207).  All in F_r, exact: every coefficient equals
// the reference's (wherever the reference can run: its NewPolZeroAt overflows a native int for n > 21, SURVEY E3).
//
// Interpolation over {1..n} in O(n log^2 n) (the domain is NOT a multiplicative subgroup, SURVEY H3):
//   1. Newton coefficients.  With y = x - 1, f(y) = sum_k d_k y(y-1)..(y-k+1) gives v_j / j! = sum_k d_k / (j-k)!,
//      i.e. (sum_j v_j/j! x^j) = (sum_k d_k x^k) e^x:   d = (v_j / j!) * e^(-x)  mod x^n  — one NTT product.
//   2. Newton -> monomial by a bottom-up divide and conquer over the subproduct tree of prod (x - i):
//        P[k0, 2s) = P[k0, s) + T[k0, s) * P[k0+s, s),   T[k0, s) = prod_{i=k0+1..k0+s} (x - i) = x^s + t(x)
//      With the leading x^s split off, t * P_R has degree <= 2s-2 and fits a cyclic size-2s transform, and the
//      merge is literally  P <- P + iNTT(NTT(pad(P_R)) . NTT(t_L))  on the whole array (P_L and x^s*P_R are already
//      in place).  The transformed t_L of every level are static per domain size and cached (QapDomain): N
//      field elements per level.  Levels with s < 16 use a schoolbook kernel, the others batched sub-transforms
//      (the last <= 10 stages of a radix-2 DIF / the first of a DIT, run on 1024-element shared-memory tiles).
//
// Included by capi.cu only.
#pragma once
#include <memory>
#include <vector>

#include "poly_host.cuh"

namespace b200 {

constexpr uint32_t kDcSchool = 16;  // merges with s < kDcSchool are schoolbook, s >= kDcSchool transform-based

// ---- batched sub-transforms --------------------------------------------------------------------------
// The last k (<= 10) stages of a DIF transform / the first k of a DIT transform only touch elements inside
// aligned blocks of 2^k: run them on contiguous 1024-element tiles in shared memory.  tw holds the plan's
// powers of w (N_plan/2 of them); tw_half = N_plan / 2.  Butterflies identical to k_ntt_dif_stage / k_ntt_dit_stage.
__global__ void __launch_bounds__(256) k_ntt_tile(Fr* __restrict__ a, const Fr* __restrict__ tw, uint32_t tw_half,
                                                  uint32_t k, int dit) {
  __shared__ Fr tile[kNttTile];
  const size_t base = (size_t)blockIdx.x * kNttTile;
  const uint32_t t = threadIdx.x;
  for (uint32_t e = t; e < kNttTile; e += blockDim.x) tile[e] = a[base + e];
  __syncthreads();
  for (uint32_t st = 0; st < k; st++) {
    const uint32_t lb = dit ? st : k - 1 - st;
    const uint32_t half = 1u << lb;
    const uint32_t stride = tw_half >> lb;
    for (uint32_t bf = t; bf < kNttTile / 2; bf += blockDim.x) {
      uint32_t j = bf & (half - 1);
      uint32_t i = ((bf - j) << 1) + j;
      Fr u = tile[i], v = tile[i + half];
      if (dit) {
        if (j) v = v * tw[(size_t)j * stride];
        tile[i] = u + v;
        tile[i + half] = u - v;
      } else {
        tile[i] = u + v;
        Fr d = u - v;
        tile[i + half] = j ? d * tw[(size_t)j * stride] : d;
      }
    }
    __syncthreads();
  }
  for (uint32_t e = t; e < kNttTile; e += blockDim.x) a[base + e] = tile[e];
}

// `total` elements = total / 2^logL independent transforms of size 2^logL on consecutive blocks.
inline cudaError_t ntt_batched(PolyCtx& pc, Fr* d, int logL, size_t total, int dit, cudaStream_t st) {
  if (logL == 0) return cudaSuccess;
  NttPlan* pl;
  PCU(pc.plan(logL, &pl, st));
  const Fr* tw = dit ? pl->tw_inv.as<Fr>() : pl->tw.as<Fr>();
  const uint32_t L_half = 1u << (logL - 1);
  const uint32_t n_half = (uint32_t)(total >> 1);
  const bool tiles = total >= kNttTile && (total % kNttTile) == 0;
  const int k_tile = tiles ? (logL < 10 ? logL : 10) : 0;
  auto upper = [&]() -> cudaError_t {   // stages with half >= 2^k_tile
    if (logL <= k_tile) return cudaSuccess;
    if (tiles && logL > 10) {           // strided shared-memory passes (ntt.cuh: k_ntt_fused), <= 8 stages each
      int up = logL - 10, top = logL - 1;
      int ks[8], hb[8], np = 0;
      while (up > 0) {
        int k = up > 8 ? 8 : up;
        ks[np] = k;
        hb[np] = top - (k - 1);
        np++;
        top -= k;
        up -= k;
      }
      for (int q = 0; q < np; q++) {
        int i = dit ? np - 1 - q : q;
        B200_LAUNCH_CTA(k_ntt_fused, (unsigned)(total / kNttTile), 256, st, d, tw, L_half, (uint32_t)hb[i], (uint32_t)ks[i], dit);
      }
      pc.note(np);
      return cudaGetLastError();
    }
    if (!dit) {
      for (uint32_t half = L_half; half >= (1u << k_tile); half >>= 1) {
        B200_LAUNCH(k_ntt_dif_stage, nblk(n_half, 256), 256, st, d, tw, n_half, half, L_half / half);
        if (half == 1) break;
      }
    } else {
      for (uint32_t half = 1u << k_tile; half <= L_half; half <<= 1)
        B200_LAUNCH(k_ntt_dit_stage, nblk(n_half, 256), 256, st, d, tw, n_half, half, L_half / half);
    }
    pc.note(logL - k_tile);
    return cudaGetLastError();
  };
  if (dit) {
    if (k_tile) { B200_LAUNCH_CTA(k_ntt_tile, (unsigned)(total / kNttTile), 256, st, d, tw, L_half, (uint32_t)k_tile, 1); pc.note(1); }
    PCU(upper());
  } else {
    PCU(upper());
    if (k_tile) { B200_LAUNCH_CTA(k_ntt_tile, (unsigned)(total / kNttTile), 256, st, d, tw, L_half, (uint32_t)k_tile, 0); pc.note(1); }
  }
  return cudaGetLastError();
}

// ---- kernels ------------------------------------------------------------------------------------------
// out[j] = sum_k val[k] * w[col[k]] over row j (CSR; val, w Montgomery)
__global__ void k_spmv_csr(const uint32_t* __restrict__ rowptr, const uint32_t* __restrict__ col,
                           const Fr* __restrict__ val, const Fr* __restrict__ w, uint32_t n, Fr* __restrict__ out) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  Fr acc = Fr::zero();
  for (uint32_t k = rowptr[j], e = rowptr[j + 1]; k < e; k++) acc = acc + val[k] * w[col[k]];
  out[j] = acc;
}
// u[j] = v[j] / j! for j < n, zero up to n_pad
__global__ void k_newton_scale(const Fr* __restrict__ v, const Fr* __restrict__ invfact, uint32_t n, uint32_t n_pad,
                               Fr* __restrict__ u) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_pad) return;
  u[j] = j < n ? v[j] * invfact[j] : Fr::zero();
}
// e[k] = (-1)^k / k! for k < n, zero up to n_pad
__global__ void k_exp_neg(const Fr* __restrict__ invfact, uint32_t n, uint32_t n_pad, Fr* __restrict__ e) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_pad) return;
  e[k] = k < n ? ((k & 1) ? invfact[k].neg() : invfact[k]) : Fr::zero();
}
// d[k] = src[k] for k < n else 0 (k < N)
__global__ void k_take(const Fr* __restrict__ src, uint32_t n, uint32_t N, Fr* __restrict__ d) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < N) d[k] = k < n ? src[k] : Fr::zero();
}
// leaves of the subproduct tree over the points offset+1 .. offset+N: t[k] = -(offset + k + 1)
__global__ void k_tree_leaves(Fr* t, uint32_t N, uint32_t offset) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= N) return;
  Fr v = Fr::zero();
  v.l[0] = offset + k + 1;
  t[k] = v.to_mont().neg();
}
// f[j] = j!  (from the inverse factorials: one inversion per element is avoided by the caller's host table)
// hv[j] = (Va[Y] * Vb[Y] * Y! - Vc[Y]) * j!   with Y = n + j,  j < n - 1   — the quotient h = (a b - c) / Z at x = Y + 1
// (a(x) = Va[Y] * Y!, Z(x) = Y! / j!); V* are the three cyclic convolutions d * (1/i!) laid out with stride M.
__global__ void k_h_values(const Fr* __restrict__ V, uint32_t M, const Fr* __restrict__ fact, uint32_t n, Fr* __restrict__ hv) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j + 1 >= n) return;
  uint32_t Y = n + j;
  Fr va = V[Y], vb = V[(size_t)M + Y], vc = V[2 * (size_t)M + Y];
  hv[j] = (va * vb * fact[Y] - vc) * fact[j];
}
// c[j] = a[j] * b[j], j < n: the values the quotient path uses in place of (C w)_j (qap_h_from_values)
__global__ void k_row_products(const Fr* __restrict__ a, const Fr* __restrict__ b, uint32_t n, Fr* __restrict__ c) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) c[j] = a[j] * b[j];
}
// schoolbook level of the tree: tc2[p*2s + i] = sum_{a+b=i} tL[a] tR[b] + (i >= s ? tL[i-s] + tR[i-s] : 0)
__global__ void k_tree_school(const Fr* __restrict__ tc, uint32_t s, uint32_t N, Fr* __restrict__ tc2) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N) return;
  uint32_t i = e & (2 * s - 1);
  const Fr* tL = tc + (e - i);
  const Fr* tR = tL + s;
  Fr acc = i >= s ? tL[i - s] + tR[i - s] : Fr::zero();
  uint32_t a_lo = i >= s ? i - s + 1 : 0, a_hi = i < s ? i : s - 1;
  for (uint32_t a = a_lo; a <= a_hi && i - a < s; a++) acc = acc + tL[a] * tR[i - a];
  tc2[e] = acc;
}
// schoolbook merge: Pout[e] = Pin[e] + sum_{a+b=i} tL[a] * PR[b]; `total` = polys * N elements, tree index = e mod N
__global__ void k_dc_school(const Fr* __restrict__ Pin, const Fr* __restrict__ tc, uint32_t s, uint32_t N,
                            uint32_t total, Fr* __restrict__ Pout) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  uint32_t i = e & (2 * s - 1);
  const Fr* PR = Pin + (e - i) + s;
  const Fr* tL = tc + ((e - i) & (N - 1));
  Fr acc = Pin[e];
  uint32_t a_lo = i >= s ? i - s + 1 : 0, a_hi = i < s ? i : s - 1;
  for (uint32_t a = a_lo; a <= a_hi; a++) acc = acc + tL[a] * PR[i - a];
  Pout[e] = acc;
}
// X[e] = i < s ? P[e + s] : 0   (the right halves, zero padded to 2s)
__global__ void k_dc_pad(const Fr* __restrict__ P, uint32_t s, uint32_t total, Fr* __restrict__ X) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  uint32_t i = e & (2 * s - 1);
  X[e] = i < s ? P[e + s] : Fr::zero();
}
// X[e] *= T[e mod N]
__global__ void k_dc_pointwise(Fr* __restrict__ X, const Fr* __restrict__ T, uint32_t N, uint32_t total) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < total) X[e] = X[e] * T[e & (N - 1)];
}
__global__ void k_add_into(Fr* __restrict__ P, const Fr* __restrict__ X, uint32_t total) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < total) P[e] = P[e] + X[e];
}
// tree build, transform level: Y[b*2s + i] = i < s ? tc[b*s + i] : 0   (every node, padded to 2s; Y has 2N elements)
__global__ void k_tree_pad(const Fr* __restrict__ tc, uint32_t s, uint32_t N, Fr* __restrict__ Y) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 2 * N) return;
  uint32_t i = e & (2 * s - 1), b = e / (2 * s);
  Y[e] = i < s ? tc[(size_t)b * s + i] : Fr::zero();
}
// from the transformed nodes Y: Tleft[p*2s+i] = Y[(2p)*2s+i] / 2s   and   W[p*2s+i] = Y[2p..] * Y[2p+1..] / 2s
__global__ void k_tree_products(const Fr* __restrict__ Y, uint32_t s, uint32_t N, Fr scale, Fr* __restrict__ Tleft,
                                Fr* __restrict__ W) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N) return;
  uint32_t i = e & (2 * s - 1), p = e / (2 * s);
  Fr l = Y[(size_t)(2 * p) * 2 * s + i] * scale;
  Tleft[e] = l;
  W[e] = l * Y[(size_t)(2 * p + 1) * 2 * s + i];
}
// tc2[e] = W[e] + (i >= s ? tL[i-s] + tR[i-s] : 0)
__global__ void k_tree_finish(const Fr* __restrict__ W, const Fr* __restrict__ tc, uint32_t s, uint32_t N,
                              Fr* __restrict__ tc2) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N) return;
  uint32_t i = e & (2 * s - 1);
  Fr v = W[e];
  if (i >= s) v = v + tc[e - s] + tc[e];   // tL[i-s] = tc[(e-i) + i-s], tR[i-s] = tc[(e-i) + s + i-s]
  tc2[e] = v;
}
// px[k] = (ab[k] - (k < n ? c[k] : 0)) for k < 2n-1; optional standard-form copy
__global__ void k_px_finish(const Fr* __restrict__ ab, const Fr* __restrict__ c, uint32_t n, Fr* __restrict__ px_mont,
                            Fr* __restrict__ px_std) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= 2 * n - 1) return;
  Fr v = ab[k];
  if (k < n) v = v - c[k];
  if (px_mont) px_mont[k] = v;
  if (px_std) px_std[k] = v.from_mont();
}
// Lagrange basis of {1..n} at tau:  l[j] = Z_n(tau) / ((tau - (j+1)) * d_j),  1/d_j = (-1)^(n-1-j) / (j! (n-1-j)!)
// zt_over[j] must hold Z_n(tau) (broadcast); tau distinct from 1..n (else flag).
__global__ void k_lagrange_at(const Fr* __restrict__ invfact, uint32_t n, Fr tau, Fr zt, Fr* __restrict__ l, int* err) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  Fr xj = Fr::zero();
  xj.l[0] = j + 1;
  Fr d = tau - xj.to_mont();
  if (d.is_zero()) {
    atomicOr(err, 16);
    l[j] = Fr::zero();
    return;
  }
  Fr v = zt * d.inverse() * invfact[j] * invfact[n - 1 - j];
  l[j] = ((n - 1 - j) & 1) ? v.neg() : v;
}

// ---- per-size domain data --------------------------------------------------------------------------------
struct QapDomain {
  size_t N = 0;                 // power of two: Newton coefficients d_0..d_{N-1}
  int logN = 0;
  DevBuf invfact;               // 1/j!, j <= nfact (Montgomery)
  DevBuf fact;                  // j! (only for the h-direct domain)
  DevBuf level[32];             // level l (s = 2^l < N): s < kDcSchool: t coefficients of every node (N elements);
                                //                        else: transformed, 1/2s-scaled t of the LEFT nodes (N elements)
  DevBuf root;                  // t of the root: prod_{i=1..N}(x - i) - x^N, N coefficients (Montgomery)
};

// offset: the tree covers the points offset+1 .. offset+N (0: the QAP domain itself; n: the points n+1.. on which the
// quotient h is interpolated directly).  nfact: factorial tables up to nfact (>= N); `fact` only when want_fact.
inline cudaError_t qap_domain_build(PolyCtx& pc, QapDomain& dom, size_t N, cudaStream_t st, size_t offset = 0, size_t nfact = 0,
                                    bool want_fact = false) {
  dom.N = N;
  dom.logN = ceil_log2(N);
  if (nfact < N) nfact = N;
  // factorials and their inverses on the host (one-time, O(nfact) multiplications)
  {
    std::vector<Fr> inv(nfact + 1), fac(want_fact ? nfact + 1 : 1);
    Fr f = Fr::one();
    if (want_fact) fac[0] = f;
    for (size_t j = 1; j <= nfact; j++) {
      f = f * fr_from_u64(j);
      if (want_fact) fac[j] = f;
    }
    Fr fi = f.inverse_impl();
    for (size_t j = nfact; j >= 1; j--) {
      inv[j] = fi;
      fi = fi * fr_from_u64(j);
    }
    inv[0] = Fr::one();
    PCU(dom.invfact.alloc((nfact + 1) * sizeof(Fr)));
    PCU(cudaMemcpyAsync(dom.invfact.p, inv.data(), (nfact + 1) * sizeof(Fr), cudaMemcpyHostToDevice, st));
    if (want_fact) {
      PCU(dom.fact.alloc((nfact + 1) * sizeof(Fr)));
      PCU(cudaMemcpyAsync(dom.fact.p, fac.data(), (nfact + 1) * sizeof(Fr), cudaMemcpyHostToDevice, st));
    }
    PCU(cudaStreamSynchronize(st));
  }
  DevBuf tcA, tcB, Y, W;
  PCU(tcA.alloc(N * sizeof(Fr)));
  PCU(tcB.alloc(N * sizeof(Fr)));
  Fr* tc = tcA.as<Fr>();
  Fr* tc2 = tcB.as<Fr>();
  B200_LAUNCH(k_tree_leaves, nblk(N, 256), 256, st, tc, (uint32_t)N, (uint32_t)offset);
  for (int l = 0; l < dom.logN; l++) {
    uint32_t s = 1u << l;
    PCU(dom.level[l].alloc(N * sizeof(Fr)));
    if (s < kDcSchool) {
      PCU(cudaMemcpyAsync(dom.level[l].p, tc, N * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
      B200_LAUNCH(k_tree_school, nblk(N, 256), 256, st, tc, s, (uint32_t)N, tc2);
    } else {
      if (!Y.p) {
        PCU(Y.alloc(2 * N * sizeof(Fr)));
        PCU(W.alloc(N * sizeof(Fr)));
      }
      B200_LAUNCH(k_tree_pad, nblk(2 * N, 256), 256, st, tc, s, (uint32_t)N, Y.as<Fr>());
      PCU(ntt_batched(pc, Y.as<Fr>(), l + 1, 2 * N, 0, st));
      NttPlan* pl;
      PCU(pc.plan(l + 1, &pl, st));
      B200_LAUNCH(k_tree_products, nblk(N, 256), 256, st, Y.as<Fr>(), s, (uint32_t)N, pl->n_inv, dom.level[l].as<Fr>(), W.as<Fr>());
      PCU(ntt_batched(pc, W.as<Fr>(), l + 1, N, 1, st));
      B200_LAUNCH(k_tree_finish, nblk(N, 256), 256, st, W.as<Fr>(), tc, s, (uint32_t)N, tc2);
    }
    Fr* tmp = tc;
    tc = tc2;
    tc2 = tmp;
  }
  PCU(dom.root.alloc(N * sizeof(Fr)));
  PCU(cudaMemcpyAsync(dom.root.p, tc, N * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
  PCU(cudaStreamSynchronize(st));   // the temporaries are freed on return
  return cudaGetLastError();
}

// In place: P holds `polys` blocks of N Newton coefficients (Montgomery); on return block q holds the N monomial
// coefficients of  sum_k d_k prod_{i=1..k} (x - i).   X: workspace of polys * N elements.
inline cudaError_t newton_to_monomial(PolyCtx& pc, const QapDomain& dom, Fr* P, Fr* X, int polys, cudaStream_t st) {
  const uint32_t N = (uint32_t)dom.N, total = (uint32_t)(dom.N * polys);
  Fr* cur = P;
  Fr* oth = X;
  for (int l = 0; l < dom.logN; l++) {
    uint32_t s = 1u << l;
    if (s < kDcSchool) {
      B200_LAUNCH(k_dc_school, nblk(total, 256), 256, st, cur, dom.level[l].as<Fr>(), s, N, total, oth);
      Fr* tmp = cur;
      cur = oth;
      oth = tmp;
      pc.note(1);
    } else {
      B200_LAUNCH(k_dc_pad, nblk(total, 256), 256, st, cur, s, total, oth);
      PCU(ntt_batched(pc, oth, l + 1, total, 0, st));
      B200_LAUNCH(k_dc_pointwise, nblk(total, 256), 256, st, oth, dom.level[l].as<Fr>(), N, total);
      PCU(ntt_batched(pc, oth, l + 1, total, 1, st));
      B200_LAUNCH(k_add_into, nblk(total, 256), 256, st, cur, oth, total);
      pc.note(3);
    }
  }
  if (cur != P) PCU(cudaMemcpyAsync(P, cur, (size_t)total * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
  return cudaGetLastError();
}

// Values v (polys blocks of `stride` elements, the first n of each used; Montgomery) at x = 1..n  ->  monomial
// coefficients in out (polys blocks of N).  ws: workspace of >= (2 * polys + 4) * N elements... see qap_workspace().
struct QapWork {
  DevBuf U, E, X;   // U: polys * 2N (Newton product operand / result), E: 2N (transformed e^-x), X: polys * N
  size_t n_e = 0, N_e = 0;   // E currently holds the series for this (n, N)
};

// Newton coefficients d (polys blocks of N, zero padded) of the values v on n consecutive integer points
inline cudaError_t newton_coeffs(PolyCtx& pc, const QapDomain& dom, QapWork& wk, const Fr* v, size_t stride, size_t n,
                                 int polys, Fr* out, cudaStream_t st) {
  const size_t N = dom.N, N2 = 2 * N;
  const int l2 = dom.logN + 1;
  PCU(wk.U.ensure(polys * N2 * sizeof(Fr)));
  PCU(wk.E.ensure(N2 * sizeof(Fr)));
  PCU(wk.X.ensure(polys * N * sizeof(Fr)));
  Fr* U = wk.U.as<Fr>();
  Fr* E = wk.E.as<Fr>();
  NttPlan* pl;
  PCU(pc.plan(l2, &pl, st));
  if (wk.n_e != n || wk.N_e != N) {   // e^(-x) mod x^n, transformed and pre-scaled by 1/2N
    B200_LAUNCH(k_exp_neg, nblk(N2, 256), 256, st, dom.invfact.as<Fr>(), (uint32_t)n, (uint32_t)N2, E);
    PCU(ntt_batched(pc, E, l2, N2, 0, st));
    B200_LAUNCH(k_scale, nblk(N2, 256), 256, st, E, (uint32_t)N2, pl->n_inv);
    wk.n_e = n;
    wk.N_e = N;
  }
  for (int q = 0; q < polys; q++)
    B200_LAUNCH(k_newton_scale, nblk(N2, 256), 256, st, v + q * stride, dom.invfact.as<Fr>(), (uint32_t)n, (uint32_t)N2, U + q * N2);
  PCU(ntt_batched(pc, U, l2, polys * N2, 0, st));
  B200_LAUNCH(k_dc_pointwise, nblk(polys * N2, 256), 256, st, U, E, (uint32_t)N2, (uint32_t)(polys * N2));
  PCU(ntt_batched(pc, U, l2, polys * N2, 1, st));
  for (int q = 0; q < polys; q++)
    B200_LAUNCH(k_take, nblk(N, 256), 256, st, U + q * N2, (uint32_t)n, (uint32_t)N, out + q * N);   // d mod x^n, padded to N
  pc.note(2 * polys + 2);
  return cudaGetLastError();
}
inline cudaError_t interpolate_ap(PolyCtx& pc, const QapDomain& dom, QapWork& wk, const Fr* v, size_t stride, size_t n,
                                  int polys, Fr* out, cudaStream_t st) {
  PCU(newton_coeffs(pc, dom, wk, v, stride, n, polys, out, st));
  return newton_to_monomial(pc, dom, out, wk.X.as<Fr>(), polys, st);
}

// ---- the quotient h = (a b - c) / Z directly from the values of a, b, c on {1..n} ------------------------------------
// GenerateProofs only consumes px through h = px / Z (groth16.go:266), and h has degree n - 2: instead of three
// interpolations (a, b, c -> coefficients), one product and one division, evaluate a, b, c on the NEXT n - 1 points
// n+1 .. 2n-1 from their Newton coefficients (a(1 + Y) / Y! = sum_k d_k / (Y - k)!: one cyclic product with the cached
// transform of 1/i! each), form h there pointwise — Z(1 + Y) = Y! / (Y - n)! — and interpolate h ONCE over the points
// n+1 .. 2n-1 (subproduct tree with offset n).  ~40 % fewer multiplications than going through px.
// This interpolates the quotient only where a b - c vanishes on 1..n.  For any witness, DivisorPolynomial drops the
// remainder, and since deg c < n = deg Z, quotient(a b - c, Z) = quotient(a b - c', Z) for c' the interpolant of the
// products a_j b_j — for which a b - c' does vanish on 1..n.  So the values of c are replaced by a_j b_j
// (qap_h_from_values) and C w is never formed: the same field elements as DivisorPolynomial(CombinePolynomials(..)) for
// satisfied and unsatisfied witnesses alike.
// The scratch of one quotient computation; a proof in flight needs its own (one per prove context).
struct QapHWork {
  QapWork work;                 // e^-x cache etc. of the final interpolation
  DevBuf V, hv, coef;           // 3 x M shift products; n-1 values of h; N' coefficients (allocated on first use)
};
// Read-only once built; its own QapHWork serves callers that compute one quotient at a time.
struct QapHDomain : QapHWork {
  size_t n = 0, M = 0;          // constraints; cyclic size of the shift products (2 * pow2 >= n)
  QapDomain tree;               // points n+1 .. n+N', factorials up to 2n
  DevBuf G;                     // transform of (1/i!)_{i < 2n-1}, size M, pre-scaled by 1/M
};
inline cudaError_t qap_hdomain_build(PolyCtx& pc, QapHDomain& hd, size_t n, cudaStream_t st) {
  hd.n = n;
  size_t N0 = 1;
  while (N0 < n) N0 <<= 1;
  hd.M = 2 * N0;
  size_t Np = 1;
  while (Np < (n > 1 ? n - 1 : 1)) Np <<= 1;
  PCU(qap_domain_build(pc, hd.tree, Np, st, n, 2 * n, true));
  PCU(hd.G.alloc(hd.M * sizeof(Fr)));
  const int lm = ceil_log2(hd.M);
  NttPlan* pl;
  PCU(pc.plan(lm, &pl, st));
  B200_LAUNCH(k_take, nblk(hd.M, 256), 256, st, hd.tree.invfact.as<Fr>(), (uint32_t)(2 * n - 1), (uint32_t)hd.M, hd.G.as<Fr>());
  PCU(ntt_batched(pc, hd.G.as<Fr>(), lm, hd.M, 0, st));
  B200_LAUNCH(k_scale, nblk(hd.M, 256), 256, st, hd.G.as<Fr>(), (uint32_t)hd.M, pl->n_inv);
  PCU(cudaStreamSynchronize(st));
  return cudaGetLastError();
}
// d: Newton coefficients of a | b | c over {1..n} (3 blocks of `dstride`, from newton_coeffs on the QAP domain);
// h_out: n - 1 coefficients of h (Montgomery) in ws->coef (ws = null: the domain's own scratch).
inline cudaError_t qap_h_from_newton(PolyCtx& pc, QapHDomain& hd, const Fr* d, size_t dstride, cudaStream_t st,
                                     QapHWork* ws = nullptr) {
  QapHWork& w = ws ? *ws : hd;
  const size_t n = hd.n, M = hd.M;
  const int lm = ceil_log2(M);
  PCU(w.V.ensure(3 * M * sizeof(Fr)));
  PCU(w.hv.ensure(n * sizeof(Fr)));
  PCU(w.coef.ensure(hd.tree.N * sizeof(Fr)));
  Fr* V = w.V.as<Fr>();
  for (int q = 0; q < 3; q++) B200_LAUNCH(k_take, nblk(M, 256), 256, st, d + q * dstride, (uint32_t)n, (uint32_t)M, V + q * M);
  PCU(ntt_batched(pc, V, lm, 3 * M, 0, st));
  B200_LAUNCH(k_dc_pointwise, nblk(3 * M, 256), 256, st, V, hd.G.as<Fr>(), (uint32_t)M, (uint32_t)(3 * M));
  PCU(ntt_batched(pc, V, lm, 3 * M, 1, st));
  if (n >= 2) {
    B200_LAUNCH(k_h_values, nblk(n - 1, 256), 256, st, V, (uint32_t)M, hd.tree.fact.as<Fr>(), (uint32_t)n, w.hv.as<Fr>());
    PCU(interpolate_ap(pc, hd.tree, w.work, w.hv.as<Fr>(), n - 1, n - 1, 1, w.coef.as<Fr>(), st));
  }
  pc.note(8);
  return cudaGetLastError();
}
// vals: the values of a | b on {1..n} in blocks 0 and 1 (n-strided, Montgomery); block 2 is overwritten with the products
// a_j b_j.  d: 3 blocks of dom.N for the Newton coefficients (dom: the QAP domain of size >= n).  h as qap_h_from_newton.
inline cudaError_t qap_h_from_values(PolyCtx& pc, const QapDomain& dom, QapWork& wk, QapHDomain& hd, Fr* vals, Fr* d,
                                     cudaStream_t st, QapHWork* ws = nullptr) {
  const size_t n = hd.n;
  B200_LAUNCH(k_row_products, nblk(n, 256), 256, st, vals, vals + n, (uint32_t)n, vals + 2 * n);
  pc.note(1);
  PCU(newton_coeffs(pc, dom, wk, vals, n, n, 3, d, st));
  return qap_h_from_newton(pc, hd, d, dom.N, st, ws);
}

// ---- a sparse R1CS resident on the device ------------------------------------------------------------------
struct SparseMat {
  DevBuf rowptr, col, val;      // CSR (n rows)
  DevBuf cptr, crow, cval;      // CSC = CSR of the transpose (m rows): the trusted setup's A^T l(tau)
  size_t nnz = 0;
};
// Witness -> px / h scratch of one proof in flight on an R1CS: one per prove context, so proofs on keys of the two
// contexts may share the R1CS and overlap.
struct R1csWork {
  DevBuf w_mont, vals, coef;        // witness (m), A w | B w | C w (3 x n; the quotient path: A w | B w | their products),
                                    // coefficients (3 x N), all Montgomery
  DevBuf px_mont;                   // 2n - 1
  DevBuf h_std;                     // h = px / Z, n - 1 coefficients, standard form (h-direct branch)
  QapWork work;
  QapHWork hw;
};
struct R1cs {
  size_t n = 0, m = 0;
  SparseMat M[3];
  DevBuf lag;                       // Lagrange basis at tau (n): the trusted setup
  std::unique_ptr<QapHDomain> hd;   // witness -> h directly (b200_groth16_prove_witness), built on first use
  std::unique_ptr<R1csWork> ws[2];  // per prove context, allocated on first use
};

}  // namespace b200
