// Batched Groth16 verification (b200_groth16_verify_batch, b200_groth16_verify_batch_device): k proofs under one Vk checked
// by ONE random linear combination,
//
//   prod_i e(rho_i A_i, B_i) * e(-(sum rho_i) alpha, beta) * e(-sum rho_i icPubl_i, gamma) * e(-sum rho_i C_i, delta) == 1,
//
// i.e. k + 3 Miller loops, one F_q^12 product and ONE final exponentiation for the whole batch, against four pairings
// per proof for k calls of groth16.VerifyProof (groth16.go:281-305).  Only *regular* proofs enter the sum — A_i, C_i on
// the curve and not infinity, B_i on the twist and in the order-r subgroup, icPubl_i not infinity, every input in range —
// and only under a regular Vk: for anything else the reference's verdict is not that of the bilinear check (it pairs a
// G1 infinity as the affine point (0, 0), bn128.go preComputeG1), so such proofs take the per-proof check (k_vb_verify_each
// in capi.cu), which is b200_groth16_verify's kernel for one proof per CTA.
//
// Launch order (capi.cu verify_batch_enqueue), a fixed sequence whatever k and whatever the outcome:
//   k_vb_classify      range, curve and subgroup tests of every proof and of the Vk -> per-proof flags
//   k_vb_ic_terms      pub_ij * IC[j+1] by the GLV half-warp product, the signals split on the device (skipped if npub = 0)
//   k_vb_ic_sum        icPubl_i = IC[0] + sum_j terms in the reference's order with its Add (as k_ic_sum)
//   k_vb_rho_terms     rho_i A_i, rho_i C_i, rho_i icPubl_i: 128-bit products, half-warp GLV routine with k2 = 0
//   k_vb_sums          G_beta, G_gamma, G_delta over the regular proofs (one CTA, complete additions)
//   k_vb_miller_warp / _thread   Miller loops of the k_reg + 3 pairs (irregular pairs contribute one)
//   k_vb_product       partial products of 64 Miller values per CTA
//   k_vb_final         product of the partials, one final exponentiation, == 1 -> aggregate bit
//   k_vb_verify_each   per-proof verdicts: regular proofs under a passed aggregate exit at once
// Host/device: tests/host/verify_batch_test.cpp runs these kernels on the CPU emulation against the oracle.
#pragma once
#include "glv.cuh"
#include "pairing_warp.cuh"

namespace b200 {
namespace vb {

constexpr uint32_t kIrregular = 1, kBad = 2;   // per-proof flags: not in the aggregate; verdict 0 without a pairing
// status word bits (include/b200snark.h)
constexpr uint32_t kStAggregate = 1, kStPerProof = 2, kStRouted = 4, kStRange = 8;
constexpr size_t kMaxBatch = (size_t)1 << 16;   // sum rho_i < 2^144 < r: the alpha scalar needs no reduction
constexpr int kMlWarps = 4;                     // warp Miller kernel: pairs per CTA
constexpr int kProdWarps = 4, kProdPerWarp = 16, kProdPerCta = kProdWarps * kProdPerWarp;
constexpr int kSumThreads = 128;

struct Vk {   // standard-form Jacobian
  Fq alpha[3];
  Fq2 beta[3], gamma[3], delta[3];
};

// proof p of a batch: 48 u64, PiA | PiC | PiB, standard-form Jacobian (b200_groth16_prove_witness_batch_device's d_out)
struct ProofView {
  const Fq* a;
  const Fq* c;
  const Fq2* b;
};
DEV ProofView proof_at(const uint64_t* proofs, size_t p) {
  const uint64_t* w = proofs + 48 * p;
  return ProofView{reinterpret_cast<const Fq*>(w), reinterpret_cast<const Fq*>(w + 12), reinterpret_cast<const Fq2*>(w + 24)};
}
template <class F>
DEV Jacobian<F> load_jac(const F* s) { return Jacobian<F>{s[0].to_mont(), s[1].to_mont(), s[2].to_mont()}; }

// Y^2 = X^3 + b Z^6 (Montgomery form)
template <class F>
DEV bool on_curve(const Jacobian<F>& p, const F& b) {
  const F z2 = p.Z.sqr(), z6 = z2.sqr() * z2;
  return p.Y.sqr() == p.X.sqr() * p.X + b * z6;
}
// a == b as group elements, neither at infinity
template <class F>
DEV bool jac_equal(const Jacobian<F>& a, const Jacobian<F>& b) {
  const F az2 = a.Z.sqr(), bz2 = b.Z.sqr();
  return a.X * bz2 == b.X * az2 && a.Y * (bz2 * b.Z) == b.Y * (az2 * a.Z);
}
// [r]Q = O for Q on the twist, not at infinity, by Scott's test for BN curves: psi(Q) == [6u^2]Q, psi the untwist-Frobenius-
// twist endomorphism of the pairing's q1 = pi(Q) (it acts on G2 as multiplication by q, and q = r + 6u^2).  Pinned against
// [r]Q = O, on and off the subgroup, by tests/test_host_verify_batch.py.
DEV bool g2_in_subgroup(const Jacobian<Fq2>& q) {
  const uint64_t k[2] = {0xf83e9682e87cfd46ULL, 0x6f4d8248eeb859fbULL};   // 6u^2, 127 bits
  Jacobian<Fq2> acc = q;
#pragma unroll 1
  for (int b = 125; b >= 0; b--) {
    acc = jac_double_ref(acc);
    if ((k[b >> 6] >> (b & 63)) & 1) acc = jac_add_complete(acc, q);
  }
  if (acc.is_inf()) return false;
  const F2 tqx = B200_F2_CONST(TWIST_MUL_BY_Q_X), tqy = B200_F2_CONST(TWIST_MUL_BY_Q_Y);
  return jac_equal(Jacobian<Fq2>{tqx * f2_conj(q.X), tqy * f2_conj(q.Y), f2_conj(q.Z)}, acc);
}
DEV bool g1_regular(const Fq* s) {
  const Jacobian<Fq> p = load_jac(s);
  const Fq three = Fq::one() + Fq::one() + Fq::one();
  return !p.is_inf() && on_curve(p, three);
}
DEV bool g2_regular(const Fq2* s) {
  const Jacobian<Fq2> q = load_jac(s);
  return !q.is_inf() && on_curve(q, B200_F2_CONST(TWIST_COEF_B)) && g2_in_subgroup(q);
}

// thread i < k: proof i; thread k: the Vk (range-checked and refused at G2 infinity on the host).  flags[i] is written
// here and only OR-ed into afterwards.
__global__ void k_vb_classify(const uint64_t* proofs, const Vk* vk, size_t k, uint32_t* flags, uint32_t* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i > k) return;
  if (i == k) {
    const bool reg = g1_regular(vk->alpha) && g2_regular(vk->beta) && g2_regular(vk->gamma) && g2_regular(vk->delta);
    flags[k] = reg ? 0 : kIrregular;
    if (!reg) atomicOr(status, kStRouted);
    return;
  }
  const ProofView v = proof_at(proofs, i);
  bool bad = false;
  for (int c = 0; c < 3; c++) bad = bad || v.a[c].geq_modulus() || v.c[c].geq_modulus() || v.b[c].geq_modulus();
  uint32_t f = 0;
  if (bad) f = kBad | kIrregular;
  else if (load_jac(v.b).is_inf()) f = kBad | kIrregular;   // the single call refuses it (the reference panics)
  else if (!(g1_regular(v.a) && g1_regular(v.c) && g2_regular(v.b))) f = kIrregular;
  flags[i] = f;
  if (f) atomicOr(status, bad ? (kStRange | kStRouted) : kStRouted);
}

// terms[i npub + j] = pub_ij * IC[j + 1], one half-warp each (k_ic_terms over a batch; the signal is GLV-split here, as the
// single call splits it on the host).  A signal >= r makes its proof bad.
__global__ void __launch_bounds__(32) k_vb_ic_terms(const Fq* ic, const uint64_t* pub, size_t npub, size_t k, Jacobian<Fq>* terms,
                                                     uint32_t* flags, uint32_t* status) {
  const uint32_t t = threadIdx.x & 31u;
  const size_t n = npub * k, j = (size_t)blockIdx.x * 2 + (t >> 4);
  const size_t jj = j < n ? j : n - 1;   // an odd count leaves the last half-warp a duplicate: every lane joins the shuffles
  const Fr v = reinterpret_cast<const Fr*>(pub)[jj];
  uint64_t kk[4] = {0, 0, 0, 0};
  uint32_t neg[2] = {0, 0};
  if (v.geq_modulus()) {
    if (j < n && (t & 15u) == 0) {
      atomicOr(flags + jj / npub, kBad | kIrregular);
      atomicOr(status, kStRange | kStRouted);
    }
  } else {
    glv_decompose(v, kk, neg);
  }
  const Jacobian<Fq> r = glv_mul_halfwarp(load_jac(ic + 3 * (jj % npub + 1)), kk, neg, t);
  if (j < n && (t & 15u) == 0) terms[j] = r;
}

// icPubl_i = IC[0] + sum_j terms, in the reference's order with its Add (k_ic_sum), standard form; infinity -> irregular
__global__ void k_vb_ic_sum(const Fq* ic, const Jacobian<Fq>* terms, size_t npub, size_t k, Fq* icp, uint32_t* flags,
                            uint32_t* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= k) return;
  Jacobian<Fq> acc = load_jac(ic);
  for (size_t j = 0; j < npub; j++) acc = jac_add_ref(acc, terms[i * npub + j]);
  icp[3 * i] = acc.X.from_mont();
  icp[3 * i + 1] = acc.Y.from_mont();
  icp[3 * i + 2] = acc.Z.from_mont();
  if (acc.is_inf()) {
    atomicOr(flags + i, kIrregular);
    atomicOr(status, kStRouted);
  }
}

// rterms[3 i + w] = rho_i * (A_i, C_i, icPubl_i)[w], one half-warp each (rho_i < 2^128: the GLV routine with k2 = 0)
__global__ void __launch_bounds__(32) k_vb_rho_terms(const uint64_t* proofs, const Fq* icp, const uint64_t* rho, size_t k,
                                                      Jacobian<Fq>* rterms) {
  const uint32_t t = threadIdx.x & 31u;
  const size_t n = 3 * k, j = (size_t)blockIdx.x * 2 + (t >> 4), jj = j < n ? j : n - 1;
  const size_t p = jj / 3;
  const ProofView v = proof_at(proofs, p);
  const Fq* src = jj % 3 == 0 ? v.a : (jj % 3 == 1 ? v.c : icp + 3 * p);
  const uint64_t kk[4] = {rho[2 * p], rho[2 * p + 1], 0, 0};
  const uint32_t neg[2] = {0, 0};
  const Jacobian<Fq> r = glv_mul_halfwarp(load_jac(src), kk, neg, t);
  if (j < n && (t & 15u) == 0) rterms[j] = r;
}

DEV void add192(uint64_t* a, const uint64_t* b) {
  unsigned __int128 c = 0;
  for (int i = 0; i < 3; i++) {
    c += (unsigned __int128)a[i] + b[i];
    a[i] = (uint64_t)c;
    c >>= 64;
  }
}
DEV Jacobian<Fq> jac_neg(const Jacobian<Fq>& p) { return Jacobian<Fq>{p.X, p.Y.neg(), p.Z}; }

// sums[0..3) = G_beta = -(sum rho_i) alpha, G_gamma = -sum rho_i icPubl_i, G_delta = -sum rho_i C_i over the regular proofs
// (none under an irregular Vk); *k_reg = their number.  One CTA: strided partial sums, then a shared-memory tree.
__global__ void __launch_bounds__(kSumThreads) k_vb_sums(const Vk* vk, const Jacobian<Fq>* rterms, const uint64_t* rho,
                                                          const uint32_t* flags, size_t k, Jacobian<Fq>* sums, uint32_t* k_reg) {
  __shared__ Jacobian<Fq> sg[kSumThreads], sd[kSumThreads];
  __shared__ uint64_t srho[kSumThreads][3];
  __shared__ uint32_t count;
  const uint32_t t = threadIdx.x;
  if (t == 0) count = 0;
  __syncthreads();
  Jacobian<Fq> g = Jacobian<Fq>::inf(), d = Jacobian<Fq>::inf();
  uint64_t s[3] = {0, 0, 0};
  uint32_t c = 0;
  if (flags[k] == 0)
    for (size_t p = t; p < k; p += kSumThreads) {
      if (flags[p]) continue;
      g = jac_add_complete(g, rterms[3 * p + 2]);
      d = jac_add_complete(d, rterms[3 * p + 1]);
      const uint64_t r3[3] = {rho[2 * p], rho[2 * p + 1], 0};
      add192(s, r3);
      c++;
    }
  sg[t] = g;
  sd[t] = d;
  for (int w = 0; w < 3; w++) srho[t][w] = s[w];
  atomicAdd(&count, c);
  __syncthreads();
  for (uint32_t h = kSumThreads / 2; h > 0; h >>= 1) {
    if (t < h) {
      sg[t] = jac_add_complete(sg[t], sg[t + h]);
      sd[t] = jac_add_complete(sd[t], sd[t + h]);
      add192(srho[t], srho[t + h]);
    }
    __syncthreads();
  }
  if (t < 32) {   // warp 0 (both halves, for the shuffles): (sum rho_i) alpha
    Fr sr = Fr::zero();
    for (int w = 0; w < 3; w++) {
      sr.l[2 * w] = (uint32_t)srho[0][w];
      sr.l[2 * w + 1] = (uint32_t)(srho[0][w] >> 32);
    }
    uint64_t kk[4];
    uint32_t neg[2];
    glv_decompose(sr, kk, neg);
    const Jacobian<Fq> r = glv_mul_halfwarp(load_jac(vk->alpha), kk, neg, t);
    if (t == 0) {
      sums[0] = jac_neg(r);
      sums[1] = jac_neg(sg[0]);
      sums[2] = jac_neg(sd[0]);
      *k_reg = count;
    }
  }
}

// the inputs of the Miller kernels
struct MlArgs {
  const uint64_t* proofs;
  const Vk* vk;
  const Jacobian<Fq>* rterms;
  const Jacobian<Fq>* sums;
  const uint32_t* flags;
  const uint32_t* k_reg;
  size_t k;
};
// pair i of the aggregate as affine Montgomery inputs: (rho_i A_i, B_i) for i < k, then (G_beta, beta), (G_gamma, gamma),
// (G_delta, delta).  false: the pair contributes one — an irregular proof, no regular proof at all, or an aggregate G1
// point at infinity (e(O, Q) = 1 is its true value; such a point is internal to the aggregate, never a reference input).
DEV bool ml_pair(const MlArgs& a, size_t i, F2::B& px, F2::B& py, F2& qx, F2& qy) {
  Jacobian<Fq> p;
  const Fq2* qs;
  if (i < a.k) {
    if (a.flags[i] || a.flags[a.k]) return false;
    p = a.rterms[3 * i];
    qs = proof_at(a.proofs, i).b;
  } else {
    if (*a.k_reg == 0) return false;
    p = a.sums[i - a.k];
    qs = i == a.k ? a.vk->beta : (i == a.k + 1 ? a.vk->gamma : a.vk->delta);
  }
  if (p.is_inf()) return false;
  const Affine<Fq> pa = jac_to_affine(p);
  const Affine<Fq2> qa = jac_to_affine(load_jac(qs));
#pragma unroll
  for (int w = 0; w < 8; w++) {
    px.l[w] = pa.x.l[w];
    py.l[w] = pa.y.l[w];
  }
  qx = qa.x;
  qy = qa.y;
  return true;
}
// one warp per pair (wp::miller_loop); mvals: six F_q^2 per pair, Montgomery form.  Args selects the pairs through its
// ml_pair overload: MlArgs above, PvbMlArgs (verify_batch_pinocchio.cuh).
template <class Args>
__global__ void __launch_bounds__(32 * kMlWarps) k_vb_miller_warp(Args a, size_t n, F2* mvals) {
  __shared__ wp::Ws wss[kMlWarps];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const size_t i = (size_t)blockIdx.x * kMlWarps + warp;
  if (i >= n) return;
  wp::Ws& ws = wss[warp];
  F2::B px, py;
  F2 qx, qy;
  int go = 0;
  if (lane == 0) go = ml_pair(a, i, px, py, qx, qy) ? 1 : 0;
  if (__shfl_sync(0xffffffffu, go, 0)) wp::miller_loop(ws, px, py, qx, qy);
  else wp::f12_set_one(ws, wp::RF);
  if (lane < 6) mvals[6 * i + lane] = ws.r[wp::RF][lane];
}
// one thread per pair (miller_loop_affine)
template <class Args>
__global__ void __launch_bounds__(32) k_vb_miller_thread(Args a, size_t n, F2* mvals) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F2::B px, py;
  F2 qx, qy;
  F12 f = F12::one();
  if (ml_pair(a, i, px, py, qx, qy)) f = miller_loop_affine(px, py, qx, qy);
  F2* o = mvals + 6 * i;
  o[0] = f.a.a; o[1] = f.a.b; o[2] = f.a.c;
  o[3] = f.b.a; o[4] = f.b.b; o[5] = f.b.c;
}

// r[0] <- prod_{b <= i < e} vals[i] (one when empty)
DEV void warp_product(wp::Ws& ws, const F2* vals, size_t b, size_t e) {
  const uint32_t lane = wp::lane_id();
  if (b >= e) {
    wp::f12_set_one(ws, 0);
    return;
  }
  if (lane < 6) ws.r[0][lane] = vals[6 * b + lane];
  wp::wsync();
  for (size_t i = b + 1; i < e; i++) {
    if (lane < 6) ws.r[1][lane] = vals[6 * i + lane];
    wp::wsync();
    wp::f12_mul(ws, 0, 0, 1);
  }
}
// warp 0's r[0] <- the product of the four warps' r[0] (two tree levels)
DEV void cta_combine(wp::Ws* wss) {
  __syncthreads();
  if ((threadIdx.x >> 5) != 0) return;
  const uint32_t lane = wp::lane_id();
  wp::Ws& ws = wss[0];
  if (lane < 6) {
    ws.r[1][lane] = wss[1].r[0][lane];
    ws.r[2][lane] = wss[2].r[0][lane];
    ws.r[3][lane] = wss[3].r[0][lane];
  }
  wp::wsync();
  wp::f12_mul(ws, 0, 0, 1);
  wp::f12_mul(ws, 2, 2, 3);
  wp::f12_mul(ws, 0, 0, 2);
}
// parts[b] = the product of Miller values [64 b, 64 b + 64)
__global__ void __launch_bounds__(32 * kProdWarps) k_vb_product(const F2* mvals, size_t n, F2* parts) {
  __shared__ wp::Ws wss[kProdWarps];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const size_t b = (size_t)blockIdx.x * kProdPerCta + (size_t)warp * kProdPerWarp;
  warp_product(wss[warp], mvals, b < n ? b : n, b + kProdPerWarp < n ? b + kProdPerWarp : n);
  cta_combine(wss);
  if (warp == 0 && lane < 6) parts[6 * blockIdx.x + lane] = wss[0].r[0][lane];
}
// the product of the partials, one final exponentiation, compared with one: *agg = 1 and status bit 0 when it is one and
// at least one proof was aggregated
__global__ void __launch_bounds__(32 * kProdWarps) k_vb_final(const F2* parts, size_t nparts, const uint32_t* k_reg, uint32_t* agg,
                                                               uint32_t* status) {
  __shared__ wp::Ws wss[kProdWarps];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const size_t per = (nparts + kProdWarps - 1) / kProdWarps, b = warp * per;
  warp_product(wss[warp], parts, b < nparts ? b : nparts, b + per < nparts ? b + per : nparts);
  cta_combine(wss);
  if (warp != 0) return;
  wp::Ws& ws = wss[0];
  wp::pairing_constants(ws);
  wp::final_exp(ws);
  const int same = lane < 6 ? (ws.r[0][lane] == (lane == 0 ? F2::one() : F2::zero()) ? 1 : 0) : 1;
  const unsigned all = __ballot_sync(0xffffffffu, same);
  if (lane == 0) {
    const bool pass = all == 0xffffffffu && *k_reg > 0;
    *agg = pass ? 1u : 0u;
    if (pass) atomicOr(status, kStAggregate);
  }
}

}  // namespace vb
}  // namespace b200
