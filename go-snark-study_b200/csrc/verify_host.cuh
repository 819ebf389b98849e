// Host-side orchestration of verification: the kernels of the single calls (b200_pairing_batch, b200_fq12_mul_batch,
// b200_groth16_verify), and the launch sequence of batched Groth16 and Pinocchio verification (verify_batch.cuh,
// verify_batch_pinocchio.cuh) over one scratch layout.  Every batch launch goes through B200_LAUNCH / B200_LAUNCH_CTA
// (poly_host.cuh), so that the SAME host code also runs in the CPU test vehicles (tests/host).  Functions return
// cudaError_t (PCU); the argument checks, with the messages b200_last_error reports, are the caller's (capi.cu).
#pragma once
#include <cstring>
#include <type_traits>
#include <vector>

#include "fixed_base.cuh"
#include "poly_host.cuh"
#include "verify_batch_pinocchio.cuh"

namespace b200 {

// ---- single calls (SURVEY §8f row 2) ----------------------------------------------------------------------------------
template <bool FAST_FE>
__device__ void pairing_from_jacobian(const Fq* g1, const Fq2* g2, F12& out, int* err) {
  bool bad = false;
  for (int k = 0; k < 3; k++) bad = bad || g1[k].geq_modulus() || g2[k].c0.geq_modulus() || g2[k].c1.geq_modulus();
  Jacobian<Fq> p{g1[0].to_mont(), g1[1].to_mont(), g1[2].to_mont()};
  Jacobian<Fq2> q{g2[0].to_mont(), g2[1].to_mont(), g2[2].to_mont()};
  if (bad || q.is_inf()) {  // G2 infinity: preComputeG2 panics "q1[2] != Fq2.One()" (bn128.go:238-241)
    atomicOr(err, bad ? 1 : 8);
    out = F12::one();
    return;
  }
  Affine<Fq> pa = jac_to_affine(p);                      // preComputeG1: G1.Affine, infinity -> (0, 0)
  Affine<Fq2> qa = jac_to_affine(q);
  F2::B px, py;
#pragma unroll
  for (int i = 0; i < 8; i++) { px.l[i] = pa.x.l[i]; py.l[i] = pa.y.l[i]; }
  out = pairing_affine_t<FAST_FE>(px, py, qa.x, qa.y);
}
__device__ void store_f12_std(const F12& f, Fq2* out) {
  out[0] = f.a.a.from_mont(); out[1] = f.a.b.from_mont(); out[2] = f.a.c.from_mont();
  out[3] = f.b.a.from_mont(); out[4] = f.b.b.from_mont(); out[5] = f.b.c.from_mont();
}
// out[i] = a[i] * b[i] in F_q^12 (fields/fq12.go:72-84), standard form in/out, [2][3][2] order
__global__ void __launch_bounds__(32) k_fq12_mul_batch(const Fq2* a, const Fq2* b, size_t n, Fq2* out, int* err) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F12 x, y;
  Fq2* xs = &x.a.a;
  Fq2* ys = &y.a.a;
  bool bad = false;
  for (int k = 0; k < 6; k++) {
    Fq2 u = a[6 * i + k], v = b[6 * i + k];
    bad = bad || u.geq_modulus() || v.geq_modulus();
    xs[k] = u.to_mont();
    ys[k] = v.to_mont();
  }
  if (bad) atomicOr(err, 1);
  store_f12_std(f12_mul(x, y), out + 6 * i);
}
template <bool FAST_FE>
__global__ void __launch_bounds__(32) k_pairing_batch(const Fq* g1, const Fq2* g2, size_t n, Fq2* out, int* err) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F12 f;
  pairing_from_jacobian<FAST_FE>(g1 + 3 * i, g2 + 3 * i, f, err);
  store_f12_std(f, out + 6 * i);
}
// one warp per pairing (pairing_warp.cuh)
constexpr int kPairWarps = 4;   // warps (pairings) per CTA: 4 x 9.5 KB of shared memory
__global__ void __launch_bounds__(32 * kPairWarps) k_pairing_batch_warp(const Fq* g1, const Fq2* g2, size_t n, Fq2* out, int* err) {
  __shared__ wp::Ws wss[kPairWarps];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const size_t i = (size_t)blockIdx.x * kPairWarps + warp;
  if (i >= n) return;
  wp::Ws& ws = wss[warp];
  F2::B px, py;
  F2 qx, qy;
  if (vb::warp_pairing_inputs(ws, g1 + 3 * i, g2 + 3 * i, px, py, qx, qy, err)) wp::pairing(ws, px, py, qx, qy);
  else wp::f12_set_one(ws, wp::RF);
  if (lane < 12) {  // standard form out, [2][3][2] order: one F_q component per lane
    const F2& c = ws.r[wp::RF][lane >> 1];
    F2::B v = ((lane & 1) ? c.c1 : c.c0).from_mont();
    Fq2* o = out + 6 * i + (lane >> 1);
    if (lane & 1) o->c1 = v;
    else o->c0 = v;
  }
}
// pts1: A, alpha1, icPubl, C ; pts2: B, beta2, gamma2, delta2 (vb::groth16_verify_cta)
__global__ void __launch_bounds__(128) k_groth16_verify(const Fq* pts1, const Fq2* pts2, int* ok, int* err) {
  __shared__ wp::Ws wss[4];
  const uint32_t warp = threadIdx.x >> 5;
  vb::groth16_verify_cta(wss, pts1 + 3 * warp, pts2 + 3 * warp, ok, err);
}
// icPubl = IC[0] + sum publicSignals[i] * IC[i+1] (groth16.go:283-286).  The products are independent: one half-warp each,
// with the GLV split of prove_host.cuh (128 doublings + ~12 additions deep instead of the 254 + ~127 of MulScalar's
// double-and-add; the same group element, which is all the pairing — it normalises its inputs — can see); the sum then runs
// in the reference's order with the reference's Add, so its degenerate cases (equal operands give Z = 0) are the reference's.
struct GlvScalar {
  uint64_t k[4];
  uint32_t neg[2];
};
__global__ void __launch_bounds__(32) k_ic_terms(const Fq* ic, const GlvScalar* gs, size_t npub, Jacobian<Fq>* terms, int* err) {
  const uint32_t t = threadIdx.x & 31u;
  const size_t i = (size_t)blockIdx.x * 2 + (t >> 4);
  const size_t ii = i < npub ? i : npub - 1;   // an odd count leaves the last half-warp a duplicate: every lane joins the shuffles
  const Fq* src = ic + 3 * (ii + 1);
  if (src[0].geq_modulus() || src[1].geq_modulus() || src[2].geq_modulus()) atomicOr(err, 1);
  Jacobian<Fq> p{src[0].to_mont(), src[1].to_mont(), src[2].to_mont()};
  GlvScalar g = gs[ii];
  Jacobian<Fq> r = glv_mul_halfwarp(p, g.k, g.neg, t);
  if (i < npub && (t & 15u) == 0) terms[i] = r;
}
__global__ void k_ic_sum(const Fq* ic, const Jacobian<Fq>* terms, size_t npub, Fq* out, int* err) {
  if (threadIdx.x | blockIdx.x) return;
  if (ic[0].geq_modulus() || ic[1].geq_modulus() || ic[2].geq_modulus()) atomicOr(err, 1);
  Jacobian<Fq> acc{ic[0].to_mont(), ic[1].to_mont(), ic[2].to_mont()};
  for (size_t i = 0; i < npub; i++) acc = jac_add_ref(acc, terms[i]);
  out[0] = acc.X.from_mont();
  out[1] = acc.Y.from_mont();
  out[2] = acc.Z.from_mont();
}

// ---- batched verification ---------------------------------------------------------------------------------------------
// What the engine takes from its caller: where launches are counted and the B200_CFG_PAIRING_KERNEL mode.
struct VbEnv {
  unsigned long long* launch_counter = nullptr;
  int pairing_kernel = 0;   // 0 auto, 1 one thread per pairing, 2 one warp per pairing
  void note(unsigned n) const { if (launch_counter) *launch_counter += n; }
  // The pairing-kernel rule of b200_pairing_batch and of both verifiers' Miller loops.  Auto: a warp per pairing has the
  // much shorter latency and wins for small calls; above 2048 pairings the thread-per-pairing kernel keeps more pairings
  // resident and has the higher throughput.
  bool thread_pairings(size_t n) const { return pairing_kernel == 1 || (pairing_kernel == 0 && n > 2048); }
};

// What a protocol's batch needs beyond the shared pipeline, by its Vk type.
template <class Vk> struct VbProto;
template <> struct VbProto<vb::Vk> {
  using MlArgs = vb::MlArgs;
  static constexpr size_t kPointFq = 3;     // per-proof G1 output of the third launch: icPubl_i
  static constexpr size_t kRhoTerms = 3;    // rho products per proof
  static constexpr size_t kSums = 3;        // aggregate G1 sums, one per fixed G2 point
  static constexpr size_t kVkThreads = 1;   // classification threads after the k proofs'
  static constexpr size_t kRhoWords = 2;    // rho words per proof
};
template <> struct VbProto<vb::PVk> {
  using MlArgs = vb::PvbMlArgs;
  static constexpr size_t kPointFq = 6;     // S_i | T_i
  static constexpr size_t kRhoTerms = vb::kPvbRhoTerms;
  static constexpr size_t kSums = vb::kPvbSums;
  static constexpr size_t kVkThreads = 7;
  static constexpr size_t kRhoWords = 10;
};

// The device image of a Vk with its IC and the batch's rho: Vk | IC | rho, standard form.
template <class Vk>
std::vector<uint8_t> vk_image(const Vk& vk, const uint64_t* ic, size_t n_ic, size_t k, const uint64_t* rho) {
  const size_t icb = n_ic * 3 * sizeof(Fq);
  std::vector<uint8_t> h(sizeof(Vk) + icb + VbProto<Vk>::kRhoWords * k * sizeof(uint64_t));
  std::memcpy(h.data(), &vk, sizeof(Vk));
  std::memcpy(h.data() + sizeof(Vk), ic, icb);
  std::memcpy(h.data() + sizeof(Vk) + icb, rho, h.size() - sizeof(Vk) - icb);
  return h;
}
inline std::vector<uint8_t> vb_vk_image(const uint64_t* ic, size_t n_ic, const uint64_t* alpha1, const uint64_t* beta2,
                                        const uint64_t* gamma2, const uint64_t* delta2, size_t k, const uint64_t* rho) {
  vb::Vk v;
  std::memcpy(v.alpha, alpha1, sizeof v.alpha);
  std::memcpy(v.beta, beta2, sizeof v.beta);
  std::memcpy(v.gamma, gamma2, sizeof v.gamma);
  std::memcpy(v.delta, delta2, sizeof v.delta);
  return vk_image(v, ic, n_ic, k, rho);
}
inline std::vector<uint8_t> pvb_vk_image(const uint64_t* ic, size_t n_ic, const uint64_t* vk_g1, const uint64_t* vk_g2, size_t k,
                                         const uint64_t* rho) {
  static_assert(sizeof(vb::PVk) == (24 + 120 + 24) * sizeof(uint64_t), "PVk is vk_g1 | vk_g2 | g2");
  vb::PVk v;
  uint8_t* w = reinterpret_cast<uint8_t*>(&v);
  std::memcpy(w, vk_g1, 24 * sizeof(uint64_t));
  std::memcpy(w + 24 * sizeof(uint64_t), vk_g2, 120 * sizeof(uint64_t));
  std::memcpy(w + 144 * sizeof(uint64_t), kG2GenJacStd, 24 * sizeof(uint64_t));
  return vk_image(v, ic, n_ic, k, rho);
}

// Per-call scratch of a batch verification, carved from one allocation.  The slots before kVbPts start every call at zero.
enum VbSlot { kVbFlags, kVbKReg, kVbAgg, kVbErr, kVbPts, kVbTerms, kVbRterms, kVbSums, kVbMvals, kVbParts, kVbSlots };
template <class Vk>
struct VbScratch {
  using P = VbProto<Vk>;
  size_t n, nparts;   // Miller pairs; partial products of k_vb_product
  size_t off[kVbSlots], bytes = 0;
  VbScratch(size_t k, size_t npub) : n(k + P::kSums), nparts((n + vb::kProdPerCta - 1) / vb::kProdPerCta) {
    const size_t sz[kVbSlots] = {(k + 1) * 4, 4, 4, 4, P::kPointFq * k * sizeof(Fq), (npub ? npub * k : 1) * sizeof(Jacobian<Fq>),
                                 P::kRhoTerms * k * sizeof(Jacobian<Fq>), P::kSums * sizeof(Jacobian<Fq>), 6 * n * sizeof(F2),
                                 6 * nparts * sizeof(F2)};
    for (int i = 0; i < kVbSlots; i++) {
      off[i] = bytes;
      bytes += (sz[i] + 255) & ~(size_t)255;
    }
  }
};

// One batch call's device inputs: the Vk image (vk_image), k proofs as the batch provers lay them out, k x npub public
// signals, the scratch (VbScratch) and the status word.
template <class Vk>
struct VbCall {
  const uint8_t* img;
  size_t n_ic;
  const uint64_t* proofs;
  const uint64_t* pub;
  size_t npub, k;
  uint8_t* scratch;
  uint32_t* status;
  const Vk* vk() const { return reinterpret_cast<const Vk*>(img); }
  const Fq* ic() const { return reinterpret_cast<const Fq*>(img + sizeof(Vk)); }
  const uint64_t* rho() const { return reinterpret_cast<const uint64_t*>(img + sizeof(Vk) + n_ic * 3 * sizeof(Fq)); }
};

// Aggregate stage, on `st`: classify -> IC terms -> per-proof sums -> rho terms -> aggregate sums -> Miller loops ->
// product -> final exponentiation (8 launches, 7 without public signals).  Zeroes the status word and the scratch's
// leading slots first; leaves the flags, the per-proof points, k_reg and agg in the scratch.
template <class Vk>
cudaError_t vb_aggregate(const VbEnv& env, const VbCall<Vk>& c, cudaStream_t st) {
  using P = VbProto<Vk>;
  constexpr bool g16 = std::is_same<Vk, vb::Vk>::value;
  const VbScratch<Vk> L(c.k, c.npub);
  const size_t k = c.k, npub = c.npub, n = L.n;
  uint32_t* flags = (uint32_t*)(c.scratch + L.off[kVbFlags]);
  uint32_t* k_reg = (uint32_t*)(c.scratch + L.off[kVbKReg]);
  uint32_t* agg = (uint32_t*)(c.scratch + L.off[kVbAgg]);
  Fq* pts = (Fq*)(c.scratch + L.off[kVbPts]);
  Jacobian<Fq>* terms = (Jacobian<Fq>*)(c.scratch + L.off[kVbTerms]);
  Jacobian<Fq>* rterms = (Jacobian<Fq>*)(c.scratch + L.off[kVbRterms]);
  Jacobian<Fq>* sums = (Jacobian<Fq>*)(c.scratch + L.off[kVbSums]);
  F2* mvals = (F2*)(c.scratch + L.off[kVbMvals]);
  F2* parts = (F2*)(c.scratch + L.off[kVbParts]);
  PCU(cudaMemsetAsync(c.scratch, 0, L.off[kVbPts], st));
  PCU(cudaMemsetAsync(c.status, 0, sizeof(uint32_t), st));
  if constexpr (g16) B200_LAUNCH(vb::k_vb_classify, nblk(k + P::kVkThreads, 64), 64, st, c.proofs, c.vk(), k, flags, c.status);
  else B200_LAUNCH(vb::k_pvb_classify, nblk(k + P::kVkThreads, 64), 64, st, c.proofs, c.vk(), k, flags, c.status);
  if (npub) B200_LAUNCH_CTA(vb::k_vb_ic_terms, nblk(npub * k, 2), 32, st, c.ic(), c.pub, npub, k, terms, flags, c.status);
  if constexpr (g16) B200_LAUNCH(vb::k_vb_ic_sum, nblk(k, 64), 64, st, c.ic(), terms, npub, k, pts, flags, c.status);
  else B200_LAUNCH(vb::k_pvb_st, nblk(k, 64), 64, st, c.ic(), terms, c.proofs, npub, k, pts, flags, c.status);
  if constexpr (g16) B200_LAUNCH_CTA(vb::k_vb_rho_terms, nblk(P::kRhoTerms * k, 2), 32, st, c.proofs, pts, c.rho(), k, rterms);
  else B200_LAUNCH_CTA(vb::k_pvb_rho_terms, nblk(P::kRhoTerms * k, 2), 32, st, c.proofs, c.vk(), pts, c.rho(), k, rterms);
  if constexpr (g16) B200_LAUNCH_CTA(vb::k_vb_sums, 1, vb::kSumThreads, st, c.vk(), rterms, c.rho(), flags, k, sums, k_reg);
  else B200_LAUNCH_CTA(vb::k_pvb_sums, vb::kPvbSums, vb::kSumThreads, st, rterms, flags, k, sums, k_reg);
  const typename P::MlArgs ma{c.proofs, c.vk(), rterms, sums, flags, k_reg, k};
  if (env.thread_pairings(n)) B200_LAUNCH(vb::k_vb_miller_thread, nblk(n, 32), 32, st, ma, n, mvals);
  else B200_LAUNCH_CTA(vb::k_vb_miller_warp, nblk(n, vb::kMlWarps), 32 * vb::kMlWarps, st, ma, n, mvals);
  B200_LAUNCH_CTA(vb::k_vb_product, (unsigned)L.nparts, 32 * vb::kProdWarps, st, mvals, n, parts);
  B200_LAUNCH_CTA(vb::k_vb_final, 1, 32 * vb::kProdWarps, st, parts, L.nparts, k_reg, agg, c.status);
  env.note(npub ? 8 : 7);
  return cudaGetLastError();
}

// Verdict stage, on `st` behind the aggregate stage: ok[0..k) the per-proof verdicts (1 launch).
template <class Vk>
cudaError_t vb_verdicts(const VbEnv& env, const VbCall<Vk>& c, int* ok, cudaStream_t st) {
  const VbScratch<Vk> L(c.k, c.npub);
  const uint32_t* flags = (const uint32_t*)(c.scratch + L.off[kVbFlags]);
  const uint32_t* agg = (const uint32_t*)(c.scratch + L.off[kVbAgg]);
  int* err = (int*)(c.scratch + L.off[kVbErr]);
  const Fq* pts = (const Fq*)(c.scratch + L.off[kVbPts]);
  if constexpr (std::is_same<Vk, vb::Vk>::value)
    B200_LAUNCH_CTA(vb::k_vb_verify_each, (unsigned)c.k, 128, st, c.proofs, c.vk(), pts, flags, agg, c.k, ok, c.status, err);
  else
    B200_LAUNCH_CTA(vb::k_pvb_verify_each, (unsigned)c.k, 128, st, c.proofs, c.vk(), pts, flags, agg, c.k, ok, c.status, err);
  env.note(1);
  return cudaGetLastError();
}

// Every launch of a batch verification: a fixed sequence whatever k and whatever the outcome, no step waits for the host.
template <class Vk>
cudaError_t verify_batch_enqueue(const VbEnv& env, const VbCall<Vk>& c, int* ok, cudaStream_t st) {
  PCU(vb_aggregate(env, c, st));
  return vb_verdicts(env, c, ok, st);
}

}  // namespace b200
