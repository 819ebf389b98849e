// Batched Pinocchio verification (b200_pinocchio_verify_batch, b200_pinocchio_verify_batch_device): k proofs under one Vk
// checked by ONE random linear combination of the five checks of snark.VerifyProof (snark.go:292-372),
//
//   1. e(PiA, Vka) e(-PiAp, g2) = 1              2. e(Vkb, PiB) e(-PiBp, g2) = 1        3. e(PiC, Vkc) e(-PiCp, g2) = 1
//   4. e(S, PiB) e(-PiH, Vkz) e(-PiC, g2) = 1    5. e(T, G2Kbg) e(G1Kbg, PiB) e(-PiKp, G2Kg) = 1
//
// with S_i = Add(Vkx_i, PiA_i), T_i = Add(S_i, PiC_i) and Vkx_i = IC[0] + sum_j pub_ij IC[j+1], all in the reference's order
// with its Add (no doubling branch: Vkx == PiA gives infinity).  Check c of proof i is raised to rho_ic (five per proof) and
// everything is multiplied together; the pairings against PiB_i merge into one per proof and each fixed G2 point collects
// one G1 sum:
//
//   prod_i e(P_i, PiB_i) * e(sum rho_i1 PiA_i, Vka) * e(sum rho_i3 PiC_i, Vkc) * e(-sum rho_i4 PiH_i, Vkz)
//     * e(sum rho_i5 T_i, G2Kbg) * e(-sum rho_i5 PiKp_i, G2Kg) * e(-sum (rho_i1 PiAp_i + rho_i2 PiBp_i + rho_i3 PiCp_i
//     + rho_i4 PiC_i), g2) == 1,     P_i = rho_i2 Vkb + rho_i4 S_i + rho_i5 G1Kbg,
//
// i.e. k_reg + 6 Miller loops, one F_q^12 product and ONE final exponentiation for the batch, against twelve pairings
// with their own final exponentiations per proof for snark.VerifyProof.  Only *regular* proofs enter the sum — the seven
// G1 points and S_i, T_i on the curve and not infinity, PiB on the twist and in the order-r subgroup, every input in range
// — and only under a regular Vk (Vkb, G1Kbg as G1 points; Vka, Vkc, G2Kbg, G2Kg, Vkz as G2 points); any other proof takes
// the per-proof check (k_pvb_verify_each below: snark.VerifyProof's twelve pairings, one CTA per proof).
//
// Launch order (verify_host.cuh: vb_aggregate, then vb_verdicts), a fixed sequence whatever k and whatever the outcome:
//   k_pvb_classify       range, curve and subgroup tests of every proof and of the Vk -> per-proof flags
//   k_vb_ic_terms        pub_ij * IC[j+1] (verify_batch.cuh; skipped if npub = 0)
//   k_pvb_st             Vkx_i, S_i, T_i in the reference's order with its Add; S_i or T_i irregular -> proof irregular
//   k_pvb_rho_terms      the 12 products of a proof by its rho_ic: 128-bit scalars, half-warp GLV routine with k2 = 0
//   k_pvb_sums           the six aggregate G1 sums over the regular proofs, one CTA per sum
//   k_vb_miller_warp / _thread   Miller loops of the k_reg + 6 pairs (PvbMlArgs; irregular pairs contribute one)
//   k_vb_product, k_vb_final     as for Groth16: product tree, one final exponentiation, == 1 -> aggregate bit
//   k_pvb_verify_each    per-proof verdicts: regular proofs under a passed aggregate exit at once
// Host/device: tests/host/pinocchio_verify_batch_test.cpp runs the classification kernel, and the aggregate through
// verify_host.cuh, on the CPU emulation against the oracle.
#pragma once
#include "verify_batch.cuh"

namespace b200 {
namespace vb {

constexpr int kPvbProofWords = 108;   // PiA, PiAp, PiBp, PiC, PiCp, PiH, PiKp (12 each), PiB (24)
constexpr int kPvbRhoTerms = 12;      // rho products per proof
constexpr int kPvbSums = 6;           // aggregate G1 sums (the fixed G2 points)
constexpr int kPvbPairings = 12;      // pairings of snark.VerifyProof

// G1 slots of a proof
enum : int { kPiA, kPiAp, kPiBp, kPiC, kPiCp, kPiH, kPiKp };

// standard-form Jacobian: vk_g1 = Vkb | G1Kbg and vk_g2 = Vka | Vkc | G2Kbg | G2Kg | Vkz as b200_pinocchio_setup returns
// them, then the G2 generator (the g2 of checks 1-4)
struct PVk {
  Fq vkb[3], g1kbg[3];
  Fq2 vka[3], vkc[3], g2kbg[3], g2kg[3], vkz[3], g2[3];
};

DEV const Fq* pvb_g1(const uint64_t* proofs, size_t p, int slot) {
  return reinterpret_cast<const Fq*>(proofs + kPvbProofWords * p + 12 * slot);
}
DEV const Fq2* pvb_b(const uint64_t* proofs, size_t p) { return reinterpret_cast<const Fq2*>(proofs + kPvbProofWords * p + 84); }

DEV void store_jac_std(Fq* o, const Jacobian<Fq>& p) {
  o[0] = p.X.from_mont();
  o[1] = p.Y.from_mont();
  o[2] = p.Z.from_mont();
}

// thread i < k: proof i; threads k .. k+6: the Vk's two G1 and five G2 points (range-checked and refused at G2 infinity
// on the host), OR-ed into flags[k].  flags is zero on entry; flags[i] is written here and only OR-ed into afterwards.
__global__ void k_pvb_classify(const uint64_t* proofs, const PVk* vk, size_t k, uint32_t* flags, uint32_t* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= k + 7) return;
  if (i >= k) {
    const int j = (int)(i - k);
    const Fq2* g2s[5] = {vk->vka, vk->vkc, vk->g2kbg, vk->g2kg, vk->vkz};
    const bool reg = j == 0 ? g1_regular(vk->vkb) : (j == 1 ? g1_regular(vk->g1kbg) : g2_regular(g2s[j - 2]));
    if (!reg) {
      atomicOr(flags + k, kIrregular);
      atomicOr(status, kStRouted);
    }
    return;
  }
  const Fq2* b = pvb_b(proofs, i);
  bool bad = false;
  for (int s = 0; s < 7; s++) {
    const Fq* g = pvb_g1(proofs, i, s);
    for (int c = 0; c < 3; c++) bad = bad || g[c].geq_modulus();
  }
  for (int c = 0; c < 3; c++) bad = bad || b[c].geq_modulus();
  uint32_t f = 0;
  if (bad || load_jac(b).is_inf()) {
    f = kBad | kIrregular;   // the host entry refuses both (the reference panics at a G2 infinity)
  } else {
    bool reg = g2_regular(b);
    for (int s = 0; s < 7; s++) reg = reg && g1_regular(pvb_g1(proofs, i, s));
    if (!reg) f = kIrregular;
  }
  flags[i] = f;
  if (f) atomicOr(status, bad ? (kStRange | kStRouted) : kStRouted);
}

// st[2 i] = S_i, st[2 i + 1] = T_i (standard-form Jacobian), with Vkx_i = IC[0] + sum_j terms in the reference's order
// and its Add, as snark.VerifyProof sums them.  S_i or T_i at infinity or off the curve (an IC point off the curve) ->
// irregular; Vkx_i itself is never paired, so its infinity is harmless.
__global__ void k_pvb_st(const Fq* ic, const Jacobian<Fq>* terms, const uint64_t* proofs, size_t npub, size_t k, Fq* st,
                         uint32_t* flags, uint32_t* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= k) return;
  Jacobian<Fq> vkx = load_jac(ic);
  for (size_t j = 0; j < npub; j++) vkx = jac_add_ref(vkx, terms[i * npub + j]);
  const Jacobian<Fq> s = jac_add_ref(vkx, load_jac(pvb_g1(proofs, i, kPiA)));
  const Jacobian<Fq> t = jac_add_ref(s, load_jac(pvb_g1(proofs, i, kPiC)));
  store_jac_std(st + 6 * i, s);
  store_jac_std(st + 6 * i + 3, t);
  const Fq three = Fq::one() + Fq::one() + Fq::one();
  if (s.is_inf() || t.is_inf() || !on_curve(s, three) || !on_curve(t, three)) {
    atomicOr(flags + i, kIrregular);
    atomicOr(status, kStRouted);
  }
}

// The 12 products of proof p, rterms[12 p + j] = rho_p[kPvbRho[j]] * (point j):
//   0 PiA rho1   1 PiC rho3   2 PiH rho4   3 T rho5   4 PiKp rho5          (the sums against Vka, Vkc, Vkz, G2Kbg, G2Kg)
//   5 PiAp rho1  6 PiBp rho2  7 PiCp rho3  8 PiC rho4                      (the sum against g2)
//   9 Vkb rho2   10 S rho4    11 G1Kbg rho5                                (P_p, paired with PiB_p)
constexpr int kSrcS = 7, kSrcT = 8, kSrcVkb = 9, kSrcKbg = 10;
// the two columns as 4-bit fields, so that a runtime index needs no local-memory table
constexpr uint64_t pack4(const int (&v)[kPvbRhoTerms]) {
  uint64_t r = 0;
  for (int j = 0; j < kPvbRhoTerms; j++) r |= (uint64_t)v[j] << (4 * j);
  return r;
}
constexpr int kPvbSrcCol[kPvbRhoTerms] = {kPiA, kPiC, kPiH, kSrcT, kPiKp, kPiAp, kPiBp, kPiCp, kPiC, kSrcVkb, kSrcS, kSrcKbg};
constexpr int kPvbRhoCol[kPvbRhoTerms] = {0, 2, 3, 4, 4, 0, 1, 2, 3, 1, 3, 4};   // c - 1 of rho_pc
constexpr uint64_t kPvbSrc = pack4(kPvbSrcCol), kPvbRho = pack4(kPvbRhoCol);
DEV int pvb_src(int j) { return (int)((kPvbSrc >> (4 * j)) & 15u); }
DEV int pvb_rho(int j) { return (int)((kPvbRho >> (4 * j)) & 15u); }
// one half-warp per product (rho < 2^128: the GLV routine with k2 = 0)
__global__ void __launch_bounds__(32) k_pvb_rho_terms(const uint64_t* proofs, const PVk* vk, const Fq* st, const uint64_t* rho,
                                                       size_t k, Jacobian<Fq>* rterms) {
  const uint32_t t = threadIdx.x & 31u;
  const size_t n = kPvbRhoTerms * k, j = (size_t)blockIdx.x * 2 + (t >> 4), jj = j < n ? j : n - 1;
  const size_t p = jj / kPvbRhoTerms;
  const int w = (int)(jj % kPvbRhoTerms), s = pvb_src(w), c = pvb_rho(w);
  const Fq* src = s < 7 ? pvb_g1(proofs, p, s)
                        : (s == kSrcS ? st + 6 * p : (s == kSrcT ? st + 6 * p + 3 : (s == kSrcVkb ? vk->vkb : vk->g1kbg)));
  const uint64_t kk[4] = {rho[10 * p + 2 * c], rho[10 * p + 2 * c + 1], 0, 0};
  const uint32_t neg[2] = {0, 0};
  const Jacobian<Fq> r = glv_mul_halfwarp(load_jac(src), kk, neg, t);
  if (j < n && (t & 15u) == 0) rterms[j] = r;
}

// CTA c of six: sums[c] over the regular proofs (none under an irregular Vk) —
//   0 sum rho1 PiA (Vka)   1 sum rho3 PiC (Vkc)   2 -sum rho4 PiH (Vkz)   3 sum rho5 T (G2Kbg)   4 -sum rho5 PiKp (G2Kg)
//   5 -sum (rho1 PiAp + rho2 PiBp + rho3 PiCp + rho4 PiC) (g2);
// CTA 0 also writes *k_reg, their number.  Strided partial sums, then k_vb_sums' shared-memory tree.
__global__ void __launch_bounds__(kSumThreads) k_pvb_sums(const Jacobian<Fq>* rterms, const uint32_t* flags, size_t k,
                                                           Jacobian<Fq>* sums, uint32_t* k_reg) {
  __shared__ Jacobian<Fq> sp[kSumThreads];
  __shared__ uint32_t count;
  const uint32_t t = threadIdx.x, c = blockIdx.x;
  if (t == 0) count = 0;
  __syncthreads();
  const int first = (int)c, last = c == kPvbSums - 1 ? 8 : (int)c;   // CTA 5 sums terms 5..8
  Jacobian<Fq> acc = Jacobian<Fq>::inf();
  uint32_t cnt = 0;
  if (flags[k] == 0)
    for (size_t p = t; p < k; p += kSumThreads) {
      if (flags[p]) continue;
      for (int j = first; j <= last; j++) acc = jac_add_complete(acc, rterms[kPvbRhoTerms * p + j]);
      cnt++;
    }
  sp[t] = acc;
  atomicAdd(&count, cnt);
  __syncthreads();
  for (uint32_t h = kSumThreads / 2; h > 0; h >>= 1) {
    if (t < h) sp[t] = jac_add_complete(sp[t], sp[t + h]);
    __syncthreads();
  }
  if (t == 0) {
    sums[c] = (c == 2 || c == 4 || c == 5) ? jac_neg(sp[0]) : sp[0];
    if (c == 0) *k_reg = count;
  }
}

// the inputs of the Miller kernels (k_vb_miller_warp / _thread over PvbMlArgs)
struct PvbMlArgs {
  const uint64_t* proofs;
  const PVk* vk;
  const Jacobian<Fq>* rterms;
  const Jacobian<Fq>* sums;
  const uint32_t* flags;
  const uint32_t* k_reg;
  size_t k;
};
// pair i of the aggregate as affine Montgomery inputs: (P_i, PiB_i) for i < k, then the six sums with Vka, Vkc, Vkz,
// G2Kbg, G2Kg, g2.  false: the pair contributes one (an irregular proof, no regular proof at all, or an aggregate G1
// point at infinity, whose true pairing is one).
DEV bool ml_pair(const PvbMlArgs& a, size_t i, F2::B& px, F2::B& py, F2& qx, F2& qy) {
  Jacobian<Fq> p;
  const Fq2* qs;
  if (i < a.k) {
    if (a.flags[i] || a.flags[a.k]) return false;
    const Jacobian<Fq>* r = a.rterms + kPvbRhoTerms * i;
    p = jac_add_complete(jac_add_complete(r[9], r[10]), r[11]);
    qs = pvb_b(a.proofs, i);
  } else {
    if (*a.k_reg == 0) return false;
    const size_t c = i - a.k;
    p = a.sums[c];
    const Fq2* g2s[kPvbSums] = {a.vk->vka, a.vk->vkc, a.vk->vkz, a.vk->g2kbg, a.vk->g2kg, a.vk->g2};
    qs = g2s[c];
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

// pairing j of snark.VerifyProof for proof p (snark.py VerifyProof's order): its G1 and G2 inputs, standard-form Jacobian
DEV const Fq* pvb_pairing_g1(const uint64_t* proofs, const PVk* vk, const Fq* st, size_t p, int j) {
  switch (j) {
    case 0: return pvb_g1(proofs, p, kPiA);
    case 1: return pvb_g1(proofs, p, kPiAp);
    case 2: return vk->vkb;
    case 3: return pvb_g1(proofs, p, kPiBp);
    case 4: return pvb_g1(proofs, p, kPiC);
    case 5: return pvb_g1(proofs, p, kPiCp);
    case 6: return st + 6 * p;
    case 7: return pvb_g1(proofs, p, kPiH);
    case 8: return pvb_g1(proofs, p, kPiC);
    case 9: return st + 6 * p + 3;
    case 10: return vk->g1kbg;
    default: return pvb_g1(proofs, p, kPiKp);
  }
}
DEV const Fq2* pvb_pairing_g2(const uint64_t* proofs, const PVk* vk, size_t p, int j) {
  switch (j) {
    case 0: return vk->vka;
    case 2: case 6: case 10: return pvb_b(proofs, p);
    case 4: return vk->vkc;
    case 7: return vk->vkz;
    case 9: return vk->g2kbg;
    case 11: return vk->g2kg;
    default: return vk->g2;
  }
}

// snark.VerifyProof over a batch, one CTA per proof: a regular proof under a passed aggregate is accepted at once, a bad one
// (coordinate >= q, signal >= r, PiB at infinity) gets 0, every other proof the reference's verdict: its twelve pairings
// (warp w runs pairings 3w .. 3w + 2 with warp_pairing_inputs' semantics), the two F_q^12 products e7 e8 and e9 e10, and
// the five comparisons of snark.go:292-372.
__global__ void __launch_bounds__(128) k_pvb_verify_each(const uint64_t* proofs, const PVk* vk, const Fq* st,
                                                         const uint32_t* flags, const uint32_t* agg, size_t k, int* ok,
                                                         uint32_t* status, int* err) {
  __shared__ wp::Ws wss[4];
  __shared__ F2 e[kPvbPairings][6];
  const size_t p = blockIdx.x;
  const uint32_t f = flags[p] | flags[k];
  if ((f & kBad) || (!f && *agg)) {
    if (threadIdx.x == 0) ok[p] = (f & kBad) ? 0 : 1;
    return;
  }
  if (threadIdx.x == 0) atomicOr(status, kStPerProof);
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  wp::Ws& ws = wss[warp];
  for (int j = 3 * (int)warp; j < 3 * (int)warp + 3; j++) {
    F2::B px, py;
    F2 qx, qy;
    if (warp_pairing_inputs(ws, pvb_pairing_g1(proofs, vk, st, p, j), pvb_pairing_g2(proofs, vk, p, j), px, py, qx, qy, err))
      wp::pairing(ws, px, py, qx, qy);
    else
      wp::f12_set_one(ws, wp::RF);
    if (lane < 6) e[j][lane] = ws.r[wp::RF][lane];
    wp::wsync();
  }
  __syncthreads();
  if (warp != 0) return;
  if (lane < 6) {
    ws.r[2][lane] = e[7][lane];
    ws.r[3][lane] = e[8][lane];
    ws.r[4][lane] = e[9][lane];
    ws.r[5][lane] = e[10][lane];
  }
  wp::wsync();
  wp::f12_mul(ws, 2, 2, 3);   // e(PiH, Vkz) e(PiC, g2)
  wp::f12_mul(ws, 4, 4, 5);   // e(T, G2Kbg) e(G1Kbg, PiB)
  int same = 1;
  if (lane < 6)
    same = e[0][lane] == e[1][lane] && e[2][lane] == e[3][lane] && e[4][lane] == e[5][lane] && e[6][lane] == ws.r[2][lane] &&
           ws.r[4][lane] == e[11][lane];
  const unsigned all = __ballot_sync(0xffffffffu, same);
  if (lane == 0) ok[p] = all == 0xffffffffu ? 1 : 0;
}

}  // namespace vb
}  // namespace b200
