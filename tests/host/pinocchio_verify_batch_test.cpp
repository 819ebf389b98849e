// CPU test vehicle for the batched Pinocchio verifier (g++, csrc/host_stub): the classification kernel and the aggregate
// kernels of verify_batch_pinocchio.cuh in the library's launch order, over emulated CTAs (one OS thread per CUDA thread,
// barriers for __syncthreads and the warp shuffles).  Test infrastructure only: never linked into libb200snark.
#include "host_stub/cuda_runtime.h"

#include <pthread.h>

#include <thread>
#include <vector>

#include "verify_batch_pinocchio.cuh"

using namespace b200;

namespace {
constexpr int kMaxWarps = 8;
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
// every CTA of a launch, one after another; the threads of a CTA run concurrently
template <class K>
void launch(unsigned nblocks, unsigned nthreads, K kernel) {
  for (unsigned b = 0; b < nblocks; b++) {
    pthread_barrier_init(&g_block_bar, nullptr, nthreads);
    for (unsigned w = 0; w < nthreads / 32; w++) pthread_barrier_init(&g_warp_bar[w], nullptr, 32);
    g_cta_mode = true;
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nthreads; t++)
      th.emplace_back([=] {
        threadIdx.x = t;
        blockIdx.x = b;
        blockDim.x = nthreads;
        gridDim.x = nblocks;
        kernel();
      });
    for (auto& x : th) x.join();
    g_cta_mode = false;
    pthread_barrier_destroy(&g_block_bar);
    for (unsigned w = 0; w < nthreads / 32; w++) pthread_barrier_destroy(&g_warp_bar[w]);
  }
}
// kernels without barriers or shuffles: one thread at a time
template <class K>
void launch_threads(unsigned nblocks, unsigned nthreads, K kernel) {
  blockDim.x = nthreads;
  gridDim.x = nblocks;
  for (unsigned b = 0; b < nblocks; b++)
    for (unsigned t = 0; t < nthreads; t++) {
      blockIdx.x = b;
      threadIdx.x = t;
      kernel();
    }
}
inline unsigned cdiv(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }
}  // namespace

extern "C" {
// k_pvb_classify over k proofs (108 u64 each: seven G1 points, PiB) and a Vk (vb::PVk: Vkb | G1Kbg | Vka | Vkc | G2Kbg |
// G2Kg | Vkz | g2, 168 u64); flags: k + 1
int t_pvb_classify(const uint64_t* proofs, const uint64_t* vk, uint32_t k, uint32_t* flags, uint32_t* status) {
  *status = 0;
  for (uint32_t i = 0; i <= k; i++) flags[i] = 0;
  launch_threads(cdiv(k + 7, 64), 64, [&] { vb::k_pvb_classify(proofs, reinterpret_cast<const vb::PVk*>(vk), k, flags, status); });
  return 0;
}
// The aggregate of a batch, kernel by kernel in pvb_enqueue's order (thread Miller kernel, warp one when warp_ml):
// flags (k + 1), st (S_i | T_i per proof, standard-form Jacobian, 24 u64 each), *agg and *status as the kernels leave
// them.  Returns k_reg.
int t_pvb_aggregate(const uint64_t* ic, const uint64_t* vk, const uint64_t* proofs, const uint64_t* pub, uint32_t npub, uint32_t k,
                    const uint64_t* rho, int warp_ml, uint32_t* flags, uint64_t* st_out, uint32_t* agg, uint32_t* status) {
  const vb::PVk* v = reinterpret_cast<const vb::PVk*>(vk);
  const Fq* dic = reinterpret_cast<const Fq*>(ic);
  const size_t n = k + vb::kPvbSums, nparts = cdiv(n, vb::kProdPerCta);
  std::vector<Jacobian<Fq>> terms(npub ? (size_t)npub * k : 1), rterms(vb::kPvbRhoTerms * (size_t)k), sums(vb::kPvbSums);
  std::vector<Fq> st(6 * (size_t)k);
  std::vector<F2> mvals(6 * n), parts(6 * nparts);
  uint32_t k_reg = 0;
  *agg = 0;
  *status = 0;
  for (uint32_t i = 0; i <= k; i++) flags[i] = 0;
  launch_threads(cdiv(k + 7, 64), 64, [&] { vb::k_pvb_classify(proofs, v, k, flags, status); });
  if (npub) launch(cdiv((size_t)npub * k, 2), 32, [&] { vb::k_vb_ic_terms(dic, pub, npub, k, terms.data(), flags, status); });
  launch_threads(cdiv(k, 64), 64, [&] { vb::k_pvb_st(dic, terms.data(), proofs, npub, k, st.data(), flags, status); });
  launch(cdiv(vb::kPvbRhoTerms * (size_t)k, 2), 32, [&] { vb::k_pvb_rho_terms(proofs, v, st.data(), rho, k, rterms.data()); });
  launch(vb::kPvbSums, vb::kSumThreads, [&] { vb::k_pvb_sums(rterms.data(), flags, k, sums.data(), &k_reg); });
  const vb::PvbMlArgs ma{proofs, v, rterms.data(), sums.data(), flags, &k_reg, k};
  if (warp_ml) launch(cdiv(n, vb::kMlWarps), 32 * vb::kMlWarps, [&] { vb::k_vb_miller_warp(ma, n, mvals.data()); });
  else launch_threads(cdiv(n, 32), 32, [&] { vb::k_vb_miller_thread(ma, n, mvals.data()); });
  launch((unsigned)nparts, 32 * vb::kProdWarps, [&] { vb::k_vb_product(mvals.data(), n, parts.data()); });
  launch(1, 32 * vb::kProdWarps, [&] { vb::k_vb_final(parts.data(), nparts, &k_reg, agg, status); });
  std::memcpy(st_out, st.data(), st.size() * sizeof(Fq));
  return (int)k_reg;
}
}
