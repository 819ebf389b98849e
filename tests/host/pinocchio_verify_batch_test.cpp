// CPU test vehicle for the batched Pinocchio verifier (g++, csrc/host_stub): the classification kernel of
// verify_batch_pinocchio.cuh, and the aggregate through the library's own engine (verify_host.cuh) on the emulated
// kernels.  Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"
#include "verify_host.cuh"

extern "C" {
// k_pvb_classify over k proofs (108 u64 each: seven G1 points, PiB) and a Vk (vb::PVk: Vkb | G1Kbg | Vka | Vkc | G2Kbg |
// G2Kg | Vkz | g2, 168 u64); flags: k + 1
int t_pvb_classify(const uint64_t* proofs, const uint64_t* vk, uint32_t k, uint32_t* flags, uint32_t* status) {
  *status = 0;
  for (uint32_t i = 0; i <= k; i++) flags[i] = 0;
  run_threads(cdiv(k + 7, 64), 64, [&] { vb::k_pvb_classify(proofs, reinterpret_cast<const vb::PVk*>(vk), k, flags, status); });
  return 0;
}
// The aggregate of a batch by the library's aggregate stage (vb_aggregate; the thread Miller kernel, the warp one when
// warp_ml) on the Vk image pvb_vk_image builds from the first 144 words of vk (its g2 is the generator): flags (k + 1),
// st (S_i | T_i per proof, standard-form Jacobian, 24 u64 each), *agg and *status as the kernels leave them.  Returns k_reg.
int t_pvb_aggregate(const uint64_t* ic, const uint64_t* vk, const uint64_t* proofs, const uint64_t* pub, uint32_t npub, uint32_t k,
                    const uint64_t* rho, int warp_ml, uint32_t* flags, uint64_t* st_out, uint32_t* agg, uint32_t* status) {
  const std::vector<uint8_t> img = pvb_vk_image(ic, npub + 1, vk, vk + 24, k, rho);
  const VbScratch<vb::PVk> L(k, npub);
  std::vector<uint8_t> s(L.bytes);
  VbEnv env;
  env.pairing_kernel = warp_ml ? 2 : 1;
  if (vb_aggregate(env, VbCall<vb::PVk>{img.data(), npub + 1, proofs, pub, npub, k, s.data(), status}, nullptr)) return -1;
  std::memcpy(flags, s.data() + L.off[kVbFlags], (k + 1) * sizeof(uint32_t));
  std::memcpy(st_out, s.data() + L.off[kVbPts], 6 * (size_t)k * sizeof(Fq));
  std::memcpy(agg, s.data() + L.off[kVbAgg], sizeof(uint32_t));
  uint32_t k_reg;
  std::memcpy(&k_reg, s.data() + L.off[kVbKReg], sizeof(uint32_t));
  return (int)k_reg;
}
}
