// Optimal-ate pairing on BN254 — the verifier side of the reference
// (bn128/bn128.go:179-421: Pairing = finalExponentiation(MillerLoop(preComputeG1, preComputeG2)),
//  fields/fq6.go, fields/fq12.go).  SURVEY §8(f) row 2.
//
// One thread per pairing (a verification is 4 independent pairings; batches of verifications are the
// GPU-shaped workload).  The tower F_q^2 -> F_q^6 = F_q^2[v]/(v^3 - (9+u)) -> F_q^12 = F_q^6[w]/(w^2 - v)
// and the line-coefficient recurrences follow the reference step by step, so the F_q^12 result is
// bit-identical to bn128.Pairing — pinned by the snarkjs golden vk_alfabeta_12 (SURVEY K8).  Like the
// reference the final exponentiation is the plain square-and-multiply by (q^12-1)/r (fq12.go:139-156);
// every intermediate is an exact field element, so any evaluation order gives the same bits.
//
// The header is host/device: tests/test_host_pairing.py runs it through the carry-flag emulation on the CPU.
#pragma once
#include "ec.cuh"
#include "pairing_constants.cuh"

namespace b200 {

using F2 = Fq2;  // outlined lazy-reduced products on the device

// constants of pairing_constants.cuh as field elements (Montgomery limbs)
#define B200_FQ_CONST(NAME) ([&] { F2::B r_; for (int i_ = 0; i_ < 8; i_++) r_.l[i_] = pc::NAME(i_); return r_; }())
#define B200_F2_CONST(NAME) (F2{B200_FQ_CONST(NAME##_0), B200_FQ_CONST(NAME##_1)})
HD F2 f2_scale(const F2& a, const F2::B& k) { return F2{a.c0 * k, a.c1 * k}; }  // Fq2.MulScalar (fq2.go:78-96)
// multiplication by the F_q^6 non-residue 9 + u  (fq6.go:31-33)
HDN F2 f2_mul_nr(const F2& a) {
  F2::B nine = B200_FQ_CONST(NINE);
  return F2{a.c0 * nine - a.c1, a.c1 * nine + a.c0};
}

struct F6 {
  F2 a, b, c;
  static HD F6 zero() { return F6{F2::zero(), F2::zero(), F2::zero()}; }
  static HD F6 one() { return F6{F2::one(), F2::zero(), F2::zero()}; }
  friend HD F6 operator+(const F6& x, const F6& y) { return F6{x.a + y.a, x.b + y.b, x.c + y.c}; }
  friend HD F6 operator-(const F6& x, const F6& y) { return F6{x.a - y.a, x.b - y.b, x.c - y.c}; }
  HD F6 neg() const { return F6{a.neg(), b.neg(), c.neg()}; }
};
// fq6.go:65-95
HDN F6 f6_mul(const F6& x, const F6& y) {
  F2 v0 = x.a * y.a, v1 = x.b * y.b, v2 = x.c * y.c;
  F2 r0 = v0 + f2_mul_nr((x.b + x.c) * (y.b + y.c) - (v1 + v2));
  F2 r1 = (x.a + x.b) * (y.a + y.b) - (v0 + v1) + f2_mul_nr(v2);
  F2 r2 = (x.a + x.c) * (y.a + y.c) - (v0 + v2) + v1;
  return F6{r0, r1, r2};
}
// multiplication by v: (a, b, c) -> (nr*c, a, b)   (fq12.go:35-41)
HD F6 f6_mul_by_v(const F6& x) { return F6{f2_mul_nr(x.c), x.a, x.b}; }

struct F12 {
  F6 a, b;
  static HD F12 one() { return F12{F6::one(), F6::zero()}; }
};
// fq12.go:72-84
HDN F12 f12_mul(const F12& x, const F12& y) {
  F6 v0 = f6_mul(x.a, y.a), v1 = f6_mul(x.b, y.b);
  return F12{v0 + f6_mul_by_v(v1), f6_mul(x.a + x.b, y.a + y.b) - (v0 + v1)};
}
// fq12.go:122-137
HDN F12 f12_sqr(const F12& x) {
  F6 ab = f6_mul(x.a, x.b);
  return F12{f6_mul(x.a + x.b, x.a + f6_mul_by_v(x.b)) - (ab + f6_mul_by_v(ab)), ab + ab};
}
// a * (ell0 + ellVV v^2... ) with the sparse element of bn128.go:402-416: b = ((ell0, 0, ellVV), (0, ellVW, 0))
HD F12 f12_mul_by_024(const F12& f, const F2& ell0, const F2& ellVW, const F2& ellVV) {
  F12 s{F6{ell0, F2::zero(), ellVV}, F6{F2::zero(), ellVW, F2::zero()}};
  return f12_mul(f, s);
}

struct EllCoeffs { F2 ell0, ellVW, ellVV; };

// bn128.go:262-294
HDN EllCoeffs pairing_doubling_step(F2& X, F2& Y, F2& Z) {
  F2::B two_inv = B200_FQ_CONST(TWO_INV);
  F2 twist_b = B200_F2_CONST(TWIST_COEF_B);
  F2 a = f2_scale(X * Y, two_inv);
  F2 b = Y.sqr();
  F2 c = Z.sqr();
  F2 d = c + (c + c);
  F2 e = twist_b * d;
  F2 f = e + (e + e);
  F2 g = f2_scale(b + f, two_inv);
  F2 h = (Y + Z).sqr() - (b + c);
  F2 i = e - b;
  F2 j = X.sqr();
  F2 e_sqr = e.sqr();
  X = a * (b - f);
  Y = g.sqr() - e_sqr - (e_sqr + e_sqr);
  Z = b * h;
  return EllCoeffs{f2_mul_nr(i), h.neg(), j + (j + j)};  // Ell0 = i * twist, twist = 9 + u
}
// bn128.go:296-330
HDN EllCoeffs pairing_mixed_addition_step(const F2& x2, const F2& y2, F2& X, F2& Y, F2& Z) {
  F2 d = X - x2 * Z;
  F2 e = Y - y2 * Z;
  F2 f = d.sqr();
  F2 g = e.sqr();
  F2 h = d * f;
  F2 i = X * f;
  F2 j = h + Z * g - (i + i);
  F2 nx = d * j;
  F2 ny = e * (i - j) - h * Y;
  F2 nz = Z * h;
  X = nx;
  Y = ny;
  Z = nz;
  return EllCoeffs{f2_mul_nr(e * x2 - d * y2), d, e.neg()};
}

// f <- f * line(P)   (the body of MillerLoop, bn128.go:360-372)
HDN F12 pairing_line(const F12& f, const EllCoeffs& c, const F2::B& px, const F2::B& py) {
  return f12_mul_by_024(f, c.ell0, f2_scale(c.ellVW, py), f2_scale(c.ellVV, px));
}

// Pairing(p1, p2) for AFFINE inputs in Montgomery form (the reference normalises first: preComputeG1 / G2.Affine).
// g2_inf: p2 is the point at infinity -> G2.Affine returns ((0,0),(1,0),(0,0)) and the reference proceeds with it.
// finalExponentiation: f^((q^12-1)/r), LSB-first square-and-multiply (fq12.go:139-156)
HDN F12 final_exp_plain(const F12& f) {
  F12 res = F12::one(), ex = f;
#pragma unroll 1
  for (int w = 0; w < pc::FINAL_EXP_WORDS; w++) {
    uint32_t word = pc::FINAL_EXP(w);
    int nbits = w == pc::FINAL_EXP_WORDS - 1 ? (2790 - 32 * (pc::FINAL_EXP_WORDS - 1)) : 32;
#pragma unroll 1
    for (int b = 0; b < nbits; b++) {
      if ((word >> b) & 1) res = f12_mul(res, ex);
      ex = f12_sqr(ex);
    }
  }
  return res;
}

// ---- the same value, ~13x fewer F_q^12 operations (EXPERIMENT: selected by the caller, off by default) ------------
// f^((q^12-1)/r) = (f^((q^6-1)(q^2+1)))^((q^4-q^2+1)/r): the easy part by one conjugation, one inversion and one
// Frobenius; the hard part by the Devegili-Scott-Dahab decomposition for BN curves (three exponentiations by the
// 63-bit parameter u and a vectorial addition chain).  It is the SAME field element as the plain exponentiation —
// pinned bit for bit on the snarkjs golden and against the plain routine (tests/test_host_pairing.py).
HDN F6 f6_inverse(const F6& x) {  // fq6.go:115-140
  F2 t0 = x.a.sqr(), t1 = x.b.sqr(), t2 = x.c.sqr();
  F2 t3 = x.a * x.b, t4 = x.a * x.c, t5 = x.b * x.c;
  F2 c0 = t0 - f2_mul_nr(t5), c1 = f2_mul_nr(t2) - t3, c2 = t1 - t4;
  F2 t6 = (x.a * c0 + f2_mul_nr(x.c * c1 + x.b * c2)).inverse();
  return F6{t6 * c0, t6 * c1, t6 * c2};
}
HDN F12 f12_inverse(const F12& x) {  // fq12.go:105-114
  F6 t2 = f6_mul(x.a, x.a) - f6_mul_by_v(f6_mul(x.b, x.b));
  F6 t3 = f6_inverse(t2);
  return F12{f6_mul(x.a, t3), f6_mul(x.b, t3).neg()};
}
HD F12 f12_conj(const F12& x) { return F12{x.a, x.b.neg()}; }  // x^(q^6)
HD F2 f2_conj(const F2& a) { return F2{a.c0, a.c1.neg()}; }
// x^(q^k), k = 1, 2, 3: in the basis 1, w, ..., w^5 (w^2 = v) the coefficient of w^j is conjugated k times and
// multiplied by xi^(j (q^k - 1) / 6)
template <int K>
HDN F12 f12_frobenius(const F12& x) {
  F2 c[6] = {x.a.a, x.b.a, x.a.b, x.b.b, x.a.c, x.b.c};
  if (K & 1) {
#pragma unroll
    for (int j = 0; j < 6; j++) c[j] = f2_conj(c[j]);
  }
  F2 g1, g2, g3, g4, g5;
  if (K == 1) {
    g1 = B200_F2_CONST(FROB1_1); g2 = B200_F2_CONST(FROB1_2); g3 = B200_F2_CONST(FROB1_3);
    g4 = B200_F2_CONST(FROB1_4); g5 = B200_F2_CONST(FROB1_5);
  } else if (K == 2) {
    g1 = B200_F2_CONST(FROB2_1); g2 = B200_F2_CONST(FROB2_2); g3 = B200_F2_CONST(FROB2_3);
    g4 = B200_F2_CONST(FROB2_4); g5 = B200_F2_CONST(FROB2_5);
  } else {
    g1 = B200_F2_CONST(FROB3_1); g2 = B200_F2_CONST(FROB3_2); g3 = B200_F2_CONST(FROB3_3);
    g4 = B200_F2_CONST(FROB3_4); g5 = B200_F2_CONST(FROB3_5);
  }
  return F12{F6{c[0], c[2] * g2, c[4] * g4}, F6{c[1] * g1, c[3] * g3, c[5] * g5}};
}
HDN F12 f12_exp_u(const F12& x) {  // x^u, MSB-first over the 63 bits of u
  F12 r = x;
#pragma unroll 1
  for (int b = 61; b >= 0; b--) {
    r = f12_sqr(r);
    if ((pc::BN_U >> b) & 1ULL) r = f12_mul(r, x);
  }
  return r;
}
HDN F12 final_exp_fast(const F12& f) {
  F12 m = f12_mul(f12_conj(f), f12_inverse(f));  // f^(q^6 - 1)
  m = f12_mul(f12_frobenius<2>(m), m);           // ^(q^2 + 1)
  F12 mu = f12_exp_u(m), mu2 = f12_exp_u(mu), mu3 = f12_exp_u(mu2);
  F12 y0 = f12_mul(f12_mul(f12_frobenius<1>(m), f12_frobenius<2>(m)), f12_frobenius<3>(m));
  F12 y1 = f12_conj(m);
  F12 y2 = f12_frobenius<2>(mu2);
  F12 y3 = f12_conj(f12_frobenius<1>(mu));
  F12 y4 = f12_conj(f12_mul(mu, f12_frobenius<1>(mu2)));
  F12 y5 = f12_conj(mu2);
  F12 y6 = f12_conj(f12_mul(mu3, f12_frobenius<1>(mu3)));
  // y0 * y1^2 * y2^6 * y3^12 * y4^18 * y5^30 * y6^36
  F12 t0 = f12_mul(f12_mul(f12_sqr(y6), y4), y5);
  F12 t1 = f12_mul(f12_mul(y3, y5), t0);
  t0 = f12_mul(t0, y2);
  t1 = f12_sqr(f12_mul(f12_sqr(t1), t0));
  t0 = f12_mul(t1, y1);
  t1 = f12_mul(t1, y0);
  return f12_mul(f12_sqr(t0), t1);
}

// MillerLoop(preComputeG1, preComputeG2) alone (bn128.go:354-398): the value pairing_affine_t exponentiates.  Miller values
// of several pairs may be multiplied before ONE final exponentiation (verify_batch.cuh).
HD F12 miller_loop_affine(const F2::B& px, const F2::B& py, const F2& qx, const F2& qy) {
  F2 X = qx, Y = qy, Z = F2::one();
  F12 f = F12::one();
  // bits of LoopCount from BitLen-2 down to 0 (bn128.go:228-236, 354-372), precompute fused with the loop
#pragma unroll 1
  for (int i = 63; i >= 0; i--) {
    EllCoeffs c = pairing_doubling_step(X, Y, Z);
    f = f12_sqr(f);
    f = pairing_line(f, c, px, py);
    if ((pc::LOOP_COUNT_LOW64 >> i) & 1) {
      c = pairing_mixed_addition_step(qx, qy, X, Y, Z);
      f = pairing_line(f, c, px, py);
    }
  }
  // q1 = pi(Q), q2 = -pi^2(Q)  (g2MulByQ on affine points: z stays one; bn128.go:238-253, 331-346)
  F2 tqx = B200_F2_CONST(TWIST_MUL_BY_Q_X), tqy = B200_F2_CONST(TWIST_MUL_BY_Q_Y);
  F2 q1x = tqx * F2{qx.c0, qx.c1.neg()}, q1y = tqy * F2{qy.c0, qy.c1.neg()};   // FrobeniusCoeffsC11 = q - 1 = -1
  F2 q2x = tqx * F2{q1x.c0, q1x.c1.neg()}, q2y = (tqy * F2{q1y.c0, q1y.c1.neg()}).neg();
  EllCoeffs c = pairing_mixed_addition_step(q1x, q1y, X, Y, Z);
  f = pairing_line(f, c, px, py);
  c = pairing_mixed_addition_step(q2x, q2y, X, Y, Z);
  return pairing_line(f, c, px, py);
}
template <bool FAST_FE>
HDN F12 pairing_affine_t(const F2::B& px, const F2::B& py, const F2& qx, const F2& qy) {
  const F12 f = miller_loop_affine(px, py, qx, qy);
  if (FAST_FE) return final_exp_fast(f);
  return final_exp_plain(f);
}
HD F12 pairing_affine(const F2::B& px, const F2::B& py, const F2& qx, const F2& qy, bool fast_final_exp = false) {
  return fast_final_exp ? pairing_affine_t<true>(px, py, qx, qy) : pairing_affine_t<false>(px, py, qx, qy);
}

}  // namespace b200
