// Short-Weierstrass group law for BN254 G1 (F = Fq) and G2 (F = Fq2), y^2 = x^3 + b.
//
// What it replaces: bn128/g1.go:32-170 and bn128/g2.go:32-200 (Jacobian
// add-2007-bl / dbl-2009-l / MSB-first double-and-add / Affine).  The kernels
// do NOT mirror those formulas: bucket accumulation uses extended-Jacobian
// "XYZZ" coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2; EFD madd-2008-s /
// add-2008-s / dbl-2008-s-1) because the mixed add costs 8M+2S against 7M+4S
// +more additions for Jacobian madd, and — unlike the reference's Add, which
// returns infinity for P+P (SURVEY H6) — every routine here handles doubling
// and inverse pairs, i.e. computes the mathematically correct sum.  Parity with
// the reference is therefore defined on affine coordinates (SURVEY H1).
//
// `Jacobian` + `jac_add_ref` / `jac_double_ref` restate the reference formulas
// themselves; they are used only by the batch scalar-mul kernel that backs
// bn128.G1/G2.MulScalar (and mints CRSs), where X,Y,Z-exact parity is testable.
#pragma once
#include "fp2.cuh"

namespace b200 {

template <class F>
struct Affine {  // (0,0) encodes the point at infinity (not on the curve: b != 0)
  F x, y;
  HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
  static HD Affine inf() { return Affine{F::zero(), F::zero()}; }
  HD Affine neg() const { return Affine{x, y.neg()}; }
};

template <class F>
struct Jacobian {  // x = X/Z^2, y = Y/Z^3, infinity <=> Z == 0 (g1.go:28-30)
  F X, Y, Z;
  HD bool is_inf() const { return Z.is_zero(); }
  static HD Jacobian inf() { return Jacobian{F::zero(), F::zero(), F::zero()}; }
};

template <class F>
struct XYZZ {  // infinity <=> ZZ == 0
  F X, Y, ZZ, ZZZ;
  HD bool is_inf() const { return ZZ.is_zero(); }
  static HD XYZZ inf() { return XYZZ{F::zero(), F::zero(), F::zero(), F::zero()}; }
  static HD XYZZ from_affine(const Affine<F>& p) {
    if (p.is_inf()) return inf();
    return XYZZ{p.x, p.y, F::one(), F::one()};
  }
  HD XYZZ neg() const { return XYZZ{X, Y.neg(), ZZ, ZZZ}; }
};

// 2*P for affine P (mdbl-2008-s-1, a = 0)
template <class F>
HD XYZZ<F> xyzz_dbl_affine(const Affine<F>& p) {
  if (p.is_inf() || p.y.is_zero()) return XYZZ<F>::inf();
  F U = p.y.dbl();
  F V = U.sqr();
  F W = U * V;
  F S = p.x * V;
  F xx = p.x.sqr();
  F M = xx.dbl() + xx;
  F X3 = M.sqr() - S.dbl();
  F Y3 = M * (S - X3) - W * p.y;
  return XYZZ<F>{X3, Y3, V, W};
}

// 2*P (dbl-2008-s-1, a = 0)
template <class F>
HD XYZZ<F> xyzz_dbl(const XYZZ<F>& p) {
  if (p.is_inf() || p.Y.is_zero()) return XYZZ<F>::inf();
  F U = p.Y.dbl();
  F V = U.sqr();
  F W = U * V;
  F S = p.X * V;
  F xx = p.X.sqr();
  F M = xx.dbl() + xx;
  F X3 = M.sqr() - S.dbl();
  F Y3 = M * (S - X3) - W * p.Y;
  return XYZZ<F>{X3, Y3, V * p.ZZ, W * p.ZZZ};
}

// acc += q, q affine (madd-2008-s), complete: handles acc = inf, q = inf,
// q = acc (doubling) and q = -acc.
template <class F>
HD void xyzz_madd(XYZZ<F>& acc, const Affine<F>& q) {
  if (q.is_inf()) return;
  if (acc.is_inf()) {
    acc = XYZZ<F>{q.x, q.y, F::one(), F::one()};
    return;
  }
  F U2 = q.x * acc.ZZ;
  F S2 = q.y * acc.ZZZ;
  F Pp = U2 - acc.X;
  F Rr = S2 - acc.Y;
  if (Pp.is_zero()) {
    if (Rr.is_zero())
      acc = xyzz_dbl_affine(q);
    else
      acc = XYZZ<F>::inf();
    return;
  }
  F PP = Pp.sqr();
  F PPP = Pp * PP;
  F Q = acc.X * PP;
  F X3 = Rr.sqr() - PPP - Q.dbl();
  F Y3 = Rr * (Q - X3) - acc.Y * PPP;
  acc.X = X3;
  acc.Y = Y3;
  acc.ZZ = acc.ZZ * PP;
  acc.ZZZ = acc.ZZZ * PPP;
}

// a += b (add-2008-s), complete.
template <class F>
HD void xyzz_add(XYZZ<F>& a, const XYZZ<F>& b) {
  if (b.is_inf()) return;
  if (a.is_inf()) {
    a = b;
    return;
  }
  F U1 = a.X * b.ZZ;
  F U2 = b.X * a.ZZ;
  F S1 = a.Y * b.ZZZ;
  F S2 = b.Y * a.ZZZ;
  F Pp = U2 - U1;
  F Rr = S2 - S1;
  if (Pp.is_zero()) {
    if (Rr.is_zero())
      a = xyzz_dbl(a);
    else
      a = XYZZ<F>::inf();
    return;
  }
  F PP = Pp.sqr();
  F PPP = Pp * PP;
  F Q = U1 * PP;
  F X3 = Rr.sqr() - PPP - Q.dbl();
  F Y3 = Rr * (Q - X3) - S1 * PPP;
  a.X = X3;
  a.Y = Y3;
  a.ZZ = a.ZZ * b.ZZ * PP;
  a.ZZZ = a.ZZZ * b.ZZZ * PPP;
}

// VT: binary-Euclid inversion (single-thread tails, where the inversion latency is the whole kernel)
template <class F, bool VT = false>
HD Affine<F> xyzz_to_affine(const XYZZ<F>& p) {
  if (p.is_inf()) return Affine<F>::inf();
  // 1/ZZZ = i ; 1/ZZ = (ZZZ * i)^2 ... cheaper: invert ZZ*ZZZ once
  F zp = p.ZZ * p.ZZZ;
  F i = VT ? zp.inverse_vartime() : zp.inverse();
  F izz = i * p.ZZZ;
  F izzz = i * p.ZZ;
  return Affine<F>{p.X * izz, p.Y * izzz};
}

// XYZZ -> Jacobian without an inversion: (X*ZZ^2, Y*ZZ^3, ZZZ) since
// ZZZ^2 = ZZ^3  =>  x = X*ZZ^2/ZZZ^2 = X/ZZ,  y = Y*ZZ^3/ZZZ^3 = Y/ZZZ.
template <class F>
HD Jacobian<F> xyzz_to_jacobian(const XYZZ<F>& p) {
  if (p.is_inf()) return Jacobian<F>::inf();
  F zz2 = p.ZZ.sqr();
  return Jacobian<F>{p.X * zz2, p.Y * (zz2 * p.ZZ), p.ZZZ};
}

// out[0..3) = the Jacobian form of p (no inversion), standard form; infinity gives three zeros
template <class F>
HD void store_jacobian_std(const XYZZ<F>& p, F* out) {
  Jacobian<F> j = xyzz_to_jacobian(p);
  out[0] = j.X.from_mont();
  out[1] = j.Y.from_mont();
  out[2] = j.Z.from_mont();
}

template <class F>
HD XYZZ<F> jacobian_to_xyzz(const Jacobian<F>& p) {
  if (p.is_inf()) return XYZZ<F>::inf();
  F zz = p.Z.sqr();
  return XYZZ<F>{p.X, p.Y, zz, zz * p.Z};
}

template <class F>
HD Affine<F> jac_to_affine(const Jacobian<F>& p) {  // g1.go:157-170
  if (p.is_inf()) return Affine<F>::inf();
  F zi = p.Z.inverse();
  F zi2 = zi.sqr();
  return Affine<F>{p.X * zi2, p.Y * (zi2 * zi)};
}

// ---- the reference's own formulas, same operation order -------------------
template <class F>
HD Jacobian<F> jac_add_ref(const Jacobian<F>& p1, const Jacobian<F>& p2) {  // g1.go:32-89
  if (p1.is_inf()) return p2;
  if (p2.is_inf()) return p1;
  F z1z1 = p1.Z.sqr();
  F z2z2 = p2.Z.sqr();
  F u1 = p1.X * z2z2;
  F u2 = p2.X * z1z1;
  F s1 = p1.Y * (p2.Z * z2z2);
  F s2 = p2.Y * (p1.Z * z1z1);
  F h = u2 - u1;
  F t2 = h + h;
  F i = t2.sqr();
  F j = h * i;
  F t3 = s2 - s1;
  F r = t3 + t3;
  F v = u1 * i;
  F x3 = r.sqr() - j - (v + v);
  F t8 = s1 * j;
  F y3 = r * (v - x3) - (t8 + t8);
  F t11 = p1.Z + p2.Z;
  F z3 = (t11.sqr() - z1z1 - z2z2) * h;
  return Jacobian<F>{x3, y3, z3};
}

template <class F>
HD Jacobian<F> jac_double_ref(const Jacobian<F>& p) {  // g1.go:101-138
  if (p.is_inf()) return p;
  F a = p.X.sqr();
  F b = p.Y.sqr();
  F c = b.sqr();
  F t0 = p.X + b;
  F d = (t0.sqr() - a - c).dbl();
  F e = a + a + a;
  F f = e.sqr();
  F x3 = f - d.dbl();
  F c2 = c + c;
  F c4 = c2 + c2;
  F y3 = e * (d - x3) - (c4 + c4);
  F z3 = (p.Y * p.Z).dbl();
  return Jacobian<F>{x3, y3, z3};
}

}  // namespace b200
