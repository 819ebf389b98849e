// Host build of the kernel arithmetic headers, for CPU unit tests only
// (tests/test_host_arith.py loads this via ctypes and compares with the
// oracle).  Not part of the product library.
#include <cstring>
#include "pairing.cuh"

using namespace b200;

namespace {
template <class F> F load(const uint32_t* p) { F r; std::memcpy(&r, p, sizeof(F)); return r; }
template <class F> void store(uint32_t* p, const F& v) { std::memcpy(p, &v, sizeof(F)); }

template <class F>
void ec_ops(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  // a: XYZZ (4 F, std form) ; b: affine (2 F) or XYZZ (4 F) ; out: affine (2 F, std form)
  constexpr int W = sizeof(F) / 4;
  XYZZ<F> A{load<F>(a).to_mont(), load<F>(a + W).to_mont(), load<F>(a + 2 * W).to_mont(), load<F>(a + 3 * W).to_mont()};
  if (op == 0) {  // madd
    Affine<F> B{load<F>(b).to_mont(), load<F>(b + W).to_mont()};
    xyzz_madd(A, B);
  } else if (op == 1) {  // add
    XYZZ<F> B{load<F>(b).to_mont(), load<F>(b + W).to_mont(), load<F>(b + 2 * W).to_mont(), load<F>(b + 3 * W).to_mont()};
    xyzz_add(A, B);
  } else if (op == 2) {
    A = xyzz_dbl(A);
  } else if (op == 3) {  // via jacobian round trip
    A = jacobian_to_xyzz(xyzz_to_jacobian(A));
  }  // op 4: none (the affine conversion by the vartime inversion)
  Affine<F> r = op == 4 ? xyzz_to_affine<F, true>(A) : xyzz_to_affine(A);
  store(out, r.x.from_mont());
  store(out + W, r.y.from_mont());
}

template <class F>
void jac_ops(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  constexpr int W = sizeof(F) / 4;
  Jacobian<F> A{load<F>(a).to_mont(), load<F>(a + W).to_mont(), load<F>(a + 2 * W).to_mont()};
  Jacobian<F> B{load<F>(b).to_mont(), load<F>(b + W).to_mont(), load<F>(b + 2 * W).to_mont()};
  Jacobian<F> r = op == 0 ? jac_add_ref(A, B) : jac_double_ref(A);
  store(out, r.X.from_mont());
  store(out + W, r.Y.from_mont());
  store(out + 2 * W, r.Z.from_mont());
}
}  // namespace

extern "C" {
// op: 0 add 1 sub 2 mul 3 inverse 4 neg 5 sqr 6 inverse_vartime ; field: 0 Fq, 1 Fr ; standard-form in/out.
// Returns 1 if the op left a Montgomery representative >= p (the conversion out of Montgomery form would hide it).
int t_fp_op(int field, int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  int noncanon = 0;
  auto run = [&](auto tag) {
    using F = decltype(tag);
    F x = load<F>(a).to_mont(), y = load<F>(b).to_mont(), r;
    switch (op) {
      case 0: r = x + y; break;
      case 1: r = x - y; break;
      case 2: r = x * y; break;
      case 3: r = x.inverse(); break;
      case 5: r = x.sqr(); break;
      case 6: r = x.inverse_vartime(); break;
      default: r = x.neg(); break;
    }
    noncanon = r.geq_modulus();
    store(out, r.from_mont());
  };
  if (field == 0) run(Fq{}); else run(Fr{});
  return noncanon;
}
// op: 0 add 1 sub 2 mul 3 inverse 4 sqr 5 neg 6 inverse_vartime ; returns 1 if a component was left >= p (as t_fp_op)
int t_fq2_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  Fq2 x = load<Fq2>(a).to_mont(), y = load<Fq2>(b).to_mont(), r;
  switch (op) {
    case 0: r = x + y; break;
    case 1: r = x - y; break;
    case 2: r = x * y; break;
    case 3: r = x.inverse(); break;
    case 4: r = x.sqr(); break;
    case 6: r = x.inverse_vartime(); break;
    default: r = x.neg(); break;
  }
  store(out, r.from_mont());
  return r.geq_modulus();
}
// w[0..16) = a * b as plain 512-bit integers (any 256-bit operands)
void t_mul_full(int k, const uint32_t* a, const uint32_t* b, uint32_t* w) {
  (void)k;
  Fq::mul_full(w, a, b);
}
// Montgomery reduction of a 512-bit value (t < p * 2^256)
void t_redc_wide(int field, int k, const uint32_t* t, uint32_t* out) {
  (void)k;
  if (field == 0) store(out, Fq::redc_wide(t));
  else store(out, Fr::redc_wide(t));
}
int t_geq(int field, const uint32_t* a) { return field == 0 ? load<Fq>(a).geq_modulus() : load<Fr>(a).geq_modulus(); }
// pairing of AFFINE standard-form inputs: g1 = (x, y), g2 = (x.c0, x.c1, y.c0, y.c1); out = 12 field elements in
// the reference's [2][3][2] order
static void pairing_common(const uint32_t* g1, const uint32_t* g2, uint32_t* out, bool fast);
void t_pairing(const uint32_t* g1, const uint32_t* g2, uint32_t* out) { pairing_common(g1, g2, out, false); }
// same pairing with the fast final exponentiation (must give the same 12 field elements)
void t_pairing_fast(const uint32_t* g1, const uint32_t* g2, uint32_t* out) { pairing_common(g1, g2, out, true); }
// F_q^12 helpers of the fast path: op 0 inverse, 1..3 Frobenius^op, 4 x^u; in/out 12 standard-form field elements
void t_f12_op(int op, const uint32_t* in, uint32_t* out) {
  F12 x;
  F2* xs[6] = {&x.a.a, &x.a.b, &x.a.c, &x.b.a, &x.b.b, &x.b.c};
  for (int k = 0; k < 6; k++) *xs[k] = load<F2>(in + 16 * k).to_mont();
  F12 r = op == 0 ? f12_inverse(x) : op == 1 ? f12_frobenius<1>(x) : op == 2 ? f12_frobenius<2>(x)
          : op == 3 ? f12_frobenius<3>(x) : f12_exp_u(x);
  const F2* parts[6] = {&r.a.a, &r.a.b, &r.a.c, &r.b.a, &r.b.b, &r.b.c};
  for (int k = 0; k < 6; k++) store(out + 16 * k, parts[k]->from_mont());
}
static void pairing_common(const uint32_t* g1, const uint32_t* g2, uint32_t* out, bool fast) {
  F2::B px = load<F2::B>(g1).to_mont(), py = load<F2::B>(g1 + 8).to_mont();
  F2 qx = load<F2>(g2).to_mont(), qy = load<F2>(g2 + 16).to_mont();
  F12 f = pairing_affine(px, py, qx, qy, fast);
  const F2* parts[6] = {&f.a.a, &f.a.b, &f.a.c, &f.b.a, &f.b.b, &f.b.c};
  for (int k = 0; k < 6; k++) store(out + 16 * k, parts[k]->from_mont());
}
void t_g1_xyzz(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) { ec_ops<Fq>(op, a, b, out); }
void t_g2_xyzz(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) { ec_ops<Fq2>(op, a, b, out); }
void t_g1_jac(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) { jac_ops<Fq>(op, a, b, out); }
void t_g2_jac(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) { jac_ops<Fq2>(op, a, b, out); }
}
