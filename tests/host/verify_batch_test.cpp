// CPU test vehicle for the batched Groth16 verifier (g++, csrc/host_stub): the split pairings (wp::miller_loop +
// wp::final_exp, miller_loop_affine + final_exp_fast), the G2 subgroup test and the classification kernel of
// verify_batch.cuh, and the aggregate through the library's own engine (verify_host.cuh) on the emulated kernels.
// Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"
#include "verify_host.cuh"

namespace {
void store_f12(uint32_t* out, const F12& f) {
  const F2* parts[6] = {&f.a.a, &f.a.b, &f.a.c, &f.b.a, &f.b.b, &f.b.c};
  for (int k = 0; k < 6; k++) store_std(out + 16 * k, *parts[k]);
}
F12 ws_f12(const wp::Ws& ws, int reg) {
  return F12{F6{ws.r[reg][0], ws.r[reg][1], ws.r[reg][2]}, F6{ws.r[reg][3], ws.r[reg][4], ws.r[reg][5]}};
}
bool f12_eq(const F12& x, const F12& y) {
  return x.a.a == y.a.a && x.a.b == y.a.b && x.a.c == y.a.c && x.b.a == y.b.a && x.b.b == y.b.b && x.b.c == y.b.c;
}
}  // namespace

extern "C" {
// One pairing of affine standard-form inputs (g1 = x, y; g2 = x.c0, x.c1, y.c0, y.c1) four ways: wp::pairing, then
// wp::miller_loop and wp::final_exp in two separate emulated launches, pairing_affine_t<true>, and miller_loop_affine +
// final_exp_fast.  out = the split warp value, 12 elements in [2][3][2] order.  Returns the number of the three other
// values that differ from it in any Montgomery word.
int t_vb_pairing_split(const uint32_t* g1, const uint32_t* g2, uint32_t* out) {
  const F2::B px = load_std<F2::B>(g1), py = load_std<F2::B>(g1 + 8);
  const F2 qx = load_std<F2>(g2), qy = load_std<F2>(g2 + 16);
  static wp::Ws ws;
  run_cta(0, 32, 1, [&] { wp::pairing(ws, px, py, qx, qy); });
  const F12 whole = ws_f12(ws, wp::RF);
  run_cta(0, 32, 1, [&] { wp::miller_loop(ws, px, py, qx, qy); });
  const F12 ml_warp = ws_f12(ws, wp::RF);
  run_cta(0, 32, 1, [&] { wp::pairing_constants(ws); wp::final_exp(ws); });
  const F12 split = ws_f12(ws, wp::RF);
  const F12 ml_thread = miller_loop_affine(px, py, qx, qy);
  store_f12(out, split);
  return !f12_eq(whole, split) + !f12_eq(pairing_affine_t<true>(px, py, qx, qy), split) +
         !f12_eq(final_exp_fast(ml_thread), split) + 10 * !f12_eq(ml_warp, ml_thread);
}
// FE(ML_1 * ML_2) for two pairs, through k_vb_product and k_vb_final's warp code; out = the value.  Returns 1 if it
// differs from pairing_1 * pairing_2 (f12_mul of two pairing_affine_t<true>).
int t_vb_fe_of_product(const uint32_t* g1a, const uint32_t* g2a, const uint32_t* g1b, const uint32_t* g2b, uint32_t* out) {
  const F2::B pxa = load_std<F2::B>(g1a), pya = load_std<F2::B>(g1a + 8), pxb = load_std<F2::B>(g1b), pyb = load_std<F2::B>(g1b + 8);
  const F2 qxa = load_std<F2>(g2a), qya = load_std<F2>(g2a + 16), qxb = load_std<F2>(g2b), qyb = load_std<F2>(g2b + 16);
  const F12 m[2] = {miller_loop_affine(pxa, pya, qxa, qya), miller_loop_affine(pxb, pyb, qxb, qyb)};
  std::vector<F2> mvals(12), parts(6);
  for (int i = 0; i < 2; i++) {
    const F2* c[6] = {&m[i].a.a, &m[i].a.b, &m[i].a.c, &m[i].b.a, &m[i].b.b, &m[i].b.c};
    for (int j = 0; j < 6; j++) mvals[6 * i + j] = *c[j];
  }
  run_cta(0, 32 * vb::kProdWarps, 1, [&] { vb::k_vb_product(mvals.data(), 2, parts.data()); });
  uint32_t k_reg = 1, agg = 0, status = 0;
  // k_vb_final only compares its value with one: the same warp code runs here on the partial to expose the value
  static wp::Ws ws;
  run_cta(0, 32, 1, [&] {
    vb::warp_product(ws, parts.data(), 0, 1);
    wp::pairing_constants(ws);
    wp::final_exp(ws);
  });
  run_cta(0, 32 * vb::kProdWarps, 1, [&] { vb::k_vb_final(parts.data(), 1, &k_reg, &agg, &status); });
  const F12 got = ws_f12(ws, 0);
  store_f12(out, got);
  const F12 want = f12_mul(pairing_affine_t<true>(pxa, pya, qxa, qya), pairing_affine_t<true>(pxb, pyb, qxb, qyb));
  const bool one = f12_eq(got, F12::one());
  return !f12_eq(got, want) + 10 * ((agg != 0) != one) + 100 * ((status & vb::kStAggregate) != 0) * !one;
}
// g2_in_subgroup on n standard-form Jacobian twist points (24 words each, on the twist, not infinity)
int t_vb_g2_subgroup(const uint32_t* q_std, uint32_t n, int* out) {
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t* s = q_std + 48 * (size_t)i;
    out[i] = vb::g2_in_subgroup(Jacobian<Fq2>{load_std<Fq2>(s), load_std<Fq2>(s + 16), load_std<Fq2>(s + 32)}) ? 1 : 0;
  }
  return 0;
}
// k_vb_classify over k proofs (48 u64 each, PiA | PiC | PiB) and a Vk (alpha | beta | gamma | delta, 12 + 3 x 24 u64)
int t_vb_classify(const uint64_t* proofs, const uint64_t* vk, uint32_t k, uint32_t* flags, uint32_t* status) {
  *status = 0;
  run_threads(cdiv(k + 1, 64), 64, [&] { vb::k_vb_classify(proofs, reinterpret_cast<const vb::Vk*>(vk), k, flags, status); });
  return 0;
}
// The aggregate of a batch by the library's aggregate stage (vb_aggregate; the thread Miller kernel, the warp one when
// warp_ml) on the Vk image vb_vk_image builds: flags (k + 1), icp (k icPubl_i, standard form, 12 u64 each), *agg and
// *status as the kernels leave them.  Returns k_reg.
int t_vb_aggregate(const uint64_t* ic, const uint64_t* vk, const uint64_t* proofs, const uint64_t* pub, uint32_t npub, uint32_t k,
                   const uint64_t* rho, int warp_ml, uint32_t* flags, uint64_t* icp_out, uint32_t* agg, uint32_t* status) {
  const std::vector<uint8_t> img = vb_vk_image(ic, npub + 1, vk, vk + 12, vk + 36, vk + 60, k, rho);
  const VbScratch<vb::Vk> L(k, npub);
  std::vector<uint8_t> s(L.bytes);
  VbEnv env;
  env.pairing_kernel = warp_ml ? 2 : 1;
  if (vb_aggregate(env, VbCall<vb::Vk>{img.data(), npub + 1, proofs, pub, npub, k, s.data(), status}, nullptr)) return -1;
  std::memcpy(flags, s.data() + L.off[kVbFlags], (k + 1) * sizeof(uint32_t));
  std::memcpy(icp_out, s.data() + L.off[kVbPts], 3 * (size_t)k * sizeof(Fq));
  std::memcpy(agg, s.data() + L.off[kVbAgg], sizeof(uint32_t));
  uint32_t k_reg;
  std::memcpy(&k_reg, s.data() + L.off[kVbKReg], sizeof(uint32_t));
  return (int)k_reg;
}
}
