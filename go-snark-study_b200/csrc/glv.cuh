// GLV scalar multiplication on BN254 G1 by the sixteen lanes of a half-warp, and the host-side lattice decomposition it
// consumes.  Used by the prover's blinding products s*A, r*B1 (groth16.go:272-273; k_groth16_products in prove_host.cuh) and
// by the verifier's public-input sum (groth16.go:283-286; k_ic_terms in verify_host.cuh).  Kept free of runtime-API calls so that the
// CPU emulation (tests/host/host_kernel_test.cpp: 32 OS threads, barrier shuffles) runs the very same lanes against the oracle.
#pragma once
#include <cstdint>
#include <cstring>

#include "ec.cuh"

namespace b200 {

// BN254's endomorphism phi(x, y) = (beta*x, y) acts as multiplication by lambda, and every k splits as k1 + k2*lambda (mod r)
// with |k1|, |k2| < 2^128 (glv_decompose below, on the host).  A 254-bit double-and-add in a lone thread is a long chain of dependent
// field multiplications and sits on the critical path of a small proof and of every verification: here sixteen lanes share
// one product (glv_mul_halfwarp).  Constants derived and checked against the oracle (tools/glv_constants.py).
struct GlvScalars {
  uint64_t k[2][4];   // product p: |k1| lo, |k1| hi, |k2| lo, |k2| hi
  uint32_t neg[2][2]; // product p: k1 < 0, k2 < 0
};

__device__ __forceinline__ Jacobian<Fq> shfl_jac(const Jacobian<Fq>& v, int lane) {
  Jacobian<Fq> r;
  const uint32_t* src = reinterpret_cast<const uint32_t*>(&v);
  uint32_t* dst = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int w = 0; w < (int)(sizeof(Jacobian<Fq>) / 4); w++) dst[w] = __shfl_sync(0xffffffffu, src[w], lane);
  return r;
}
// complete addition on top of the reference formula (which has no doubling branch); G1 and G2
template <class F>
__device__ Jacobian<F> jac_add_complete(const Jacobian<F>& a, const Jacobian<F>& b) {
  if (a.is_inf()) return b;
  if (b.is_inf()) return a;
  Jacobian<F> r = jac_add_ref(a, b);
  if (r.Z.is_zero()) {  // same x: either a == b (double) or a == -b (infinity)
    F z1z1 = a.Z.sqr(), z2z2 = b.Z.sqr();
    if (a.Y * (b.Z * z2z2) == b.Y * (a.Z * z1z1)) return jac_double_ref(a);
    return Jacobian<F>::inf();
  }
  return r;
}

// k * P by the sixteen lanes of a half-warp (lanes t with the same t >> 4; ALL 32 lanes of the warp must call).  k1 = k[0..1],
// k2 = k[2..3], signs in neg[0..1].  Lanes 0..7 of the half take the eight 16-bit chunks of |k1| on P and lanes 8..15 those of
// |k2| on phi(P): a chunk is 16 doublings + <= 16 additions, lane q then shifts by 16 q doublings, and a 3-level shuffle tree
// + one addition join the sixteen partial products.  Depth: 128 Jacobian doublings + ~12 additions (the doublings are the
// floor of any double-and-add on a 128-bit GLV half), against 128 + ~36 with four 64-bit chunks.  The product is returned
// in the half's first lane (t & 15 == 0); P at infinity or k = 0 give the point at infinity.
__device__ Jacobian<Fq> glv_mul_halfwarp(Jacobian<Fq> p, const uint64_t k[4], const uint32_t neg[2], uint32_t t) {
  const uint32_t half = (t >> 3) & 1u, q = t & 7u;
  if (half) {  // phi(P): x -> beta * x
    Fq beta;
    const uint32_t bm[8] = {0xd782e155u, 0x71930c11u, 0xffbe3323u, 0xa6bb947cu, 0xd4741444u, 0xaa303344u, 0x26594943u, 0x2c3b3f0du};
#pragma unroll
    for (int i = 0; i < 8; i++) beta.l[i] = bm[i];
    p.X = p.X * beta;
  }
  if (neg[half]) p.Y = p.Y.neg();
  const uint64_t word = k[2 * half + (q >> 2)];
  const uint32_t chunk = (uint32_t)(word >> (16 * (q & 3u))) & 0xffffu;
  Jacobian<Fq> r = Jacobian<Fq>::inf();
  bool started = false;
  for (int b = 15; b >= 0; b--) {
    uint32_t bit = (chunk >> b) & 1u;
    if (!started && !bit) continue;
    started = true;
    r = jac_double_ref(r);
    if (bit) r = jac_add_ref(r, p);   // r = m*p with m >= 2 or infinity: never equal to +-p
  }
  if (started)
    for (uint32_t d = 0; d < 16 * q; d++) r = jac_double_ref(r);   // * 2^(16 q)
  const uint32_t base8 = t & ~7u;
#pragma unroll
  for (int off = 4; off > 0; off >>= 1) {
    Jacobian<Fq> other = shfl_jac(r, (int)(base8 + ((q + off) & 7u)));
    if ((int)q < off) r = jac_add_complete(r, other);
  }
  Jacobian<Fq> k2part = shfl_jac(r, (int)((t & ~15u) + 8));
  if ((t & 15u) == 0) r = jac_add_complete(r, k2part);
  return r;
}

// k = k1 + k2*lambda (mod r), |k1|, |k2| < 2^128.  Lattice basis of BN254's GLV endomorphism:
//   a1 = 0x89d3256894d213e3, b1 = -0x6f4d8248eeb859fc8211bbeb7d4f1128, a2 = 0x6f4d8248eeb859fd0be4e1541221250b, b2 = a1
// c1 = round(b2*k/r), c2 = round(-b1*k/r) through g_i = round(2^256 * |.| / r);  k1 = k - c1*a1 - c2*a2,  k2 = c1*|b1| - c2*b2.
// Any rounding error only lengthens k1, k2 by a bit; k1 + k2*lambda == k holds by construction.  Host and device: the
// batch verifier splits public signals that are already in device memory (verify_batch.cuh).
struct U5 { uint64_t l[5]; };
HD U5 u5_mul(const uint64_t* a, int na, const uint64_t* b, int nb) {  // (na + nb <= 5 significant limbs)
  uint64_t t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < na; i++) {
    unsigned __int128 c = 0;
    for (int j = 0; j < nb; j++) {
      c += (unsigned __int128)a[i] * b[j] + t[i + j];
      t[i + j] = (uint64_t)c;
      c >>= 64;
    }
    t[i + nb] += (uint64_t)c;
  }
  U5 r;
  for (int i = 0; i < 5; i++) r.l[i] = t[i];
  return r;
}
HD U5 u5_sub(const U5& a, const U5& b) {
  U5 r;
  unsigned __int128 br = 0;
  for (int i = 0; i < 5; i++) {
    unsigned __int128 d = (unsigned __int128)a.l[i] - b.l[i] - (uint64_t)br;
    r.l[i] = (uint64_t)d;
    br = (d >> 64) & 1;
  }
  return r;
}
HD bool u5_abs(U5& a) {  // two's complement -> magnitude; returns the sign
  bool neg = (a.l[4] >> 63) != 0;
  if (neg) {
    unsigned __int128 c = 1;
    for (int i = 0; i < 5; i++) {
      c += (uint64_t)~a.l[i];
      a.l[i] = (uint64_t)c;
      c >>= 64;
    }
  }
  return neg;
}
HD int glv_decompose(const Fr& k_std, uint64_t out[4], uint32_t neg[2]) {
  const uint64_t A1[2] = {0x89d3256894d213e3ULL, 0}, B1m[2] = {0x8211bbeb7d4f1128ULL, 0x6f4d8248eeb859fcULL};
  const uint64_t A2[2] = {0x0be4e1541221250bULL, 0x6f4d8248eeb859fdULL}, B2[2] = {0x89d3256894d213e3ULL, 0};
  const uint64_t G1c[3] = {0xd91d232ec7e0b3d7ULL, 0x2ULL, 0}, G2c[3] = {0x7a7bd9d4391eb18eULL, 0x4ccef014a773d2cfULL, 0x2ULL};
  uint64_t k[4];
  memcpy(k, &k_std, 32);
  auto round_shift = [&](const uint64_t* g, uint64_t c[3]) {  // (k * g + 2^255) >> 256
    uint64_t t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) {
      unsigned __int128 cy = 0;
      for (int j = 0; j < 3; j++) {
        cy += (unsigned __int128)k[i] * g[j] + t[i + j];
        t[i + j] = (uint64_t)cy;
        cy >>= 64;
      }
      t[i + 3] += (uint64_t)cy;
    }
    unsigned __int128 cy = (unsigned __int128)t[3] + 0x8000000000000000ULL;
    cy >>= 64;
    for (int i = 4; i < 7; i++) {
      cy += t[i];
      c[i - 4] = (uint64_t)cy;
      cy >>= 64;
    }
  };
  uint64_t c1[3], c2[3];
  round_shift(G1c, c1);
  round_shift(G2c, c2);
  U5 kk{{k[0], k[1], k[2], k[3], 0}};
  U5 k1 = u5_sub(u5_sub(kk, u5_mul(c1, 3, A1, 1)), u5_mul(c2, 3, A2, 2));
  U5 k2 = u5_sub(u5_mul(c1, 3, B1m, 2), u5_mul(c2, 3, B2, 1));
  neg[0] = u5_abs(k1);
  neg[1] = u5_abs(k2);
  if (k1.l[2] | k1.l[3] | k1.l[4] | k2.l[2] | k2.l[3] | k2.l[4]) return -1;  // cannot happen (|k_i| < 2^128)
  out[0] = k1.l[0]; out[1] = k1.l[1]; out[2] = k2.l[0]; out[3] = k2.l[1];
  return 0;
}

}  // namespace b200
