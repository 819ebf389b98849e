// Fixed-base batch scalar multiplication: out[i] = k_i * G for one generator G (the G1 or the G2 generator) and n
// scalars in device memory — the minting step of the trusted setup (groth16/groth16.go:139-220, snark.go:171-248
// call G.MulScalar(generator, k) once per CRS point).
//
// The reference-order kernel k_mul_batch_ref walks all 254 bits with a data-dependent add, to stay X,Y,Z-exact with
// the reference.  A setup only needs the same group elements (parity is on affine coordinates), so here every thread
// recodes its scalar into signed c-bit digits (for_each_digit, the MSM's recode) and adds +-T[w][|d|-1] from a table
// T[w][d-1] = d * 2^(c*w) * G with XYZZ mixed additions: ceil(255/c) additions and no doublings per point.  The table
// is the MSM window table (window_table_enqueue) of the base set {1*G, 2*G, .., 2^(c-1)*G}, built per call.
//
// The host code launches through B200_LAUNCH (poly_host.cuh), so the CPU test vehicle (tests/host) runs this same
// orchestration over the emulated kernels.
#pragma once
#include <vector>

#include "msm.cuh"
#include "poly_host.cuh"

namespace b200 {

// Window bits of the fixed-base kernel.  With c = 12 the G1 table is 22 windows x 2048 points x 64 B = 2.75 MiB and the
// G2 table 5.5 MiB, both resident in the H100's 50 MB L2.  Kernel time at 2^20 for c = 8 / 10 / 12: DESIGN.md §4.
#ifndef B200_FIXED_BASE_C
#define B200_FIXED_BASE_C 12
#endif
constexpr int kFixedBaseC = B200_FIXED_BASE_C;
constexpr uint32_t kFixedBaseWin = (255 + kFixedBaseC - 1) / kFixedBaseC;
constexpr uint32_t kFixedBaseRow = 1u << (kFixedBaseC - 1);   // table points per window

// Generators in standard-form Jacobian limbs (bn128/bn128.go:52-83).
inline const uint64_t kG1GenJacStd[12] = {1, 0, 0, 0, 2, 0, 0, 0, 1, 0, 0, 0};
inline const uint64_t kG2GenJacStd[24] = {
    0x46debd5cd992f6edull, 0x674322d4f75edaddull, 0x426a00665e5c4479ull, 0x1800deef121f1e76ull,
    0x97e485b7aef312c2ull, 0xf1aa493335a9e712ull, 0x7260bfb731fb5d25ull, 0x198e9393920d483aull,
    0x4ce6cc0166fa7daaull, 0xe3d1e7690c43d37bull, 0x4aab71808dcb408full, 0x12c85ea5db8c6debull,
    0x55acdadcd122975bull, 0xbc4b313370b38ef3ull, 0xec9e99ad690c3395ull, 0x090689d0585ff075ull,
    1, 0, 0, 0, 0, 0, 0, 0};

// table[w][i] = 2^(c*w) * P_i (Montgomery affine) for w < nwin, from n standard-form Jacobian points on the device, or,
// with jac_std null, from the points already in row 0 (minted there by fixed_base_row_enqueue).  state: n XYZZ records of
// scratch.  err |= 1 when a coordinate is >= q.  (The window precompute of an MSM base set.)
template <class F>
void window_table_enqueue(const F* jac_std, size_t n, uint32_t nwin, int c, Affine<F>* table, XYZZ<F>* state, int* err,
                          cudaStream_t st) {
  auto* to_affine = &k_batch_to_affine<F, 8>;
  if (jac_std) B200_LAUNCH(k_load_bases<F>, nblk(n, 128), 128, st, jac_std, n, table, err);
  B200_LAUNCH(k_affine_to_xyzz<F>, nblk(n, 128), 128, st, table, state, n);
  for (uint32_t w = 1; w < nwin; w++) {
    B200_LAUNCH(k_window_step<F>, nblk(n, 128), 128, st, state, n, c);
    B200_LAUNCH(to_affine, nblk((n + 7) / 8, 128), 128, st, state, table + (size_t)w * n, n);
  }
}

// acc = k_i * G: one thread per scalar (standard form, < r), signed digits of kFixedBaseC bits, one mixed addition per
// non-zero digit.  Scalar 0 gives the XYZZ infinity.
template <class F>
__global__ void __launch_bounds__(128) k_fixed_base(const Affine<F>* __restrict__ table, const Fr* __restrict__ scalars,
                                                    size_t n, XYZZ<F>* __restrict__ out) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr v = ld_fe(&scalars[i]);
  constexpr MsmShape sh{0, (uint32_t)kFixedBaseC, kFixedBaseWin, kFixedBaseRow, kFixedBaseRow};
  XYZZ<F> acc = XYZZ<F>::inf();
  for_each_digit(v.l, sh, [&](uint32_t w, uint32_t d, uint32_t neg) {
    Affine<F> p = ld_affine(&table[w * kFixedBaseRow + d - 1]);
    if (neg) p.y = p.y.neg();
    xyzz_madd(acc, p);
  });
  out[i] = acc;
}

// Montgomery affine -> standard-form Jacobian (x, y, 1), infinity -> all zero (k_finalize's writer, one thread per point).
template <class F>
__global__ void k_affine_store_std(const Affine<F>* __restrict__ in, size_t n, F* __restrict__ out_jac_std) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<F> a = in[i];
  F* o = out_jac_std + 3 * i;
  if (a.is_inf()) {
    o[0] = F::zero();
    o[1] = F::zero();
    o[2] = F::zero();
    return;
  }
  o[0] = a.x.from_mont();
  o[1] = a.y.from_mont();
  F one = F::zero();
  reinterpret_cast<uint32_t*>(&one)[0] = 1;
  o[2] = one;
}

// The generator table of k_fixed_base for F's group: kFixedBaseWin x kFixedBaseRow affine points (2.75 MiB in G1,
// 5.5 MiB in G2), built once per call and shared by every set that call mints.
template <class F>
struct FixedBaseTable {
  DevBuf table;
  // the base set {1*G, .., 2^(c-1)*G}, then its window table.  err |= 1 if a coordinate were >= q (never, for the generators)
  cudaError_t build(int* err, cudaStream_t st) {
    constexpr size_t H = kFixedBaseRow;
    const uint64_t* gen = sizeof(F) == sizeof(Fq) ? kG1GenJacStd : kG2GenJacStd;
    std::vector<Fr> ks(H);
    for (size_t d = 0; d < H; d++) {
      ks[d] = Fr::zero();
      ks[d].l[0] = (uint32_t)(d + 1);
    }
    DevBuf dgen, dks, base, state;
    PCU(dgen.alloc(3 * sizeof(F)));
    PCU(dks.alloc(H * sizeof(Fr)));
    PCU(base.alloc(3 * H * sizeof(F)));
    PCU(state.alloc(H * sizeof(XYZZ<F>)));
    PCU(table.alloc((size_t)kFixedBaseWin * H * sizeof(Affine<F>)));
    PCU(cudaMemcpyAsync(dgen.p, gen, 3 * sizeof(F), cudaMemcpyHostToDevice, st));
    PCU(cudaMemcpyAsync(dks.p, ks.data(), H * sizeof(Fr), cudaMemcpyHostToDevice, st));
    B200_LAUNCH(k_mul_batch_ref<F>, nblk(H, 128), 128, st, dgen.as<F>(), 1, dks.as<Fr>(), H, base.as<F>(), err);
    window_table_enqueue<F>(base.as<F>(), H, kFixedBaseWin, kFixedBaseC, table.as<Affine<F>>(), state.as<XYZZ<F>>(), err, st);
    PCU(cudaGetLastError());
    return cudaStreamSynchronize(st);   // the temporaries above are freed on return
  }
};

// row0[i] = scalars[i] * G as Montgomery affine points, infinity as Affine::inf() (the words k_load_bases writes for the
// same points), for n standard-form scalars < r on the device.  state: n XYZZ records of scratch.  row0 is row 0 of a
// base set's table (setup into a resident key) or a plain buffer (fixed_base_mul).
template <class F>
void fixed_base_row_enqueue(const FixedBaseTable<F>& gen, const Fr* d_scalars_std, size_t n, Affine<F>* row0,
                            XYZZ<F>* state, cudaStream_t st) {
  if (n == 0) return;
  auto* to_affine = &k_batch_to_affine<F, 8>;
  B200_LAUNCH(k_fixed_base<F>, nblk(n, 128), 128, st, gen.table.template as<Affine<F>>(), d_scalars_std, n, state);
  B200_LAUNCH(to_affine, nblk((n + 7) / 8, 128), 128, st, state, row0, n);
}

// out_jac_std[i] = scalars[i] * G under a built generator table: affine (x, y, 1) in standard form, infinity all zero,
// stored from the minted row.  Returns after synchronising `st`.
template <class F>
cudaError_t fixed_base_std(const FixedBaseTable<F>& gen, const Fr* d_scalars_std, size_t n, F* d_out_jac_std, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  DevBuf state, aff;
  PCU(state.alloc(n * sizeof(XYZZ<F>)));
  PCU(aff.alloc(n * sizeof(Affine<F>)));
  fixed_base_row_enqueue<F>(gen, d_scalars_std, n, aff.as<Affine<F>>(), state.as<XYZZ<F>>(), st);
  B200_LAUNCH(k_affine_store_std<F>, nblk(n, 128), 128, st, aff.as<Affine<F>>(), n, d_out_jac_std);
  PCU(cudaGetLastError());
  return cudaStreamSynchronize(st);
}

// out_jac_std[i] = scalars[i] * G (G the generator of F's group) for n standard-form scalars < r on the device; affine
// (x, y, 1) in standard form, infinity all zero.  Builds the generator table, mints and stores; returns after
// synchronising `st`.  err |= 1 if a table coordinate were >= q (never, for the generators).
template <class F>
cudaError_t fixed_base_mul(const Fr* d_scalars_std, size_t n, F* d_out_jac_std, int* err, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  FixedBaseTable<F> gen;
  PCU(gen.build(err, st));
  return fixed_base_std<F>(gen, d_scalars_std, n, d_out_jac_std, st);
}

}  // namespace b200
