// Device build of the kernel arithmetic headers, for the on-device edge tests only (tests/test_gpu_arith.py loads it via
// ctypes and compares with the oracle).  The twin of tests/host/host_arith_test.cpp: the same operations under the same
// op numbers, but compiled by nvcc for sm_90a, so the carry chains are the PTX condition-code chains ptxas fuses, the
// INL = true variants are the force-inlined products of the hot kernels and the INL = false ones the __noinline__
// outlined products of the cold kernels.  Not part of the product library.
//
// Every entry point takes n operands in host arrays of 32-bit limbs (standard form; the kernels convert to and from
// Montgomery form), runs ONE kernel launch over all of them, synchronises, and returns the CUDA error code.
#include <cuda_runtime.h>

#include <cstring>
#include <vector>

#include "glv.cuh"
#include "pairing_warp.cuh"

using namespace b200;

namespace {

struct DevBuf {
  void* p = nullptr;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  template <class T> T* as() const { return static_cast<T*>(p); }
};

#define TRY(x)                                  \
  do {                                          \
    cudaError_t e_ = (x);                       \
    if (e_ != cudaSuccess) return (int)e_;      \
  } while (0)

cudaError_t upload(DevBuf& b, const void* h, size_t bytes) {
  cudaError_t e = cudaMalloc(&b.p, bytes ? bytes : 1);
  if (e != cudaSuccess || !h) return e;
  return cudaMemcpy(b.p, h, bytes, cudaMemcpyHostToDevice);
}
// the launch has been issued: pick up its error, wait for it, copy the result back
int finish(void* h_out, const DevBuf& d_out, size_t bytes) {
  TRY(cudaGetLastError());
  TRY(cudaDeviceSynchronize());
  TRY(cudaMemcpy(h_out, d_out.p, bytes, cudaMemcpyDeviceToHost));
  return 0;
}
unsigned blocks(size_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

template <class F> __device__ __forceinline__ F ld(const uint32_t* p) {
  F r;
  uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int k = 0; k < (int)(sizeof(F) / 4); k++) d[k] = p[k];
  return r;
}
template <class F> __device__ __forceinline__ void st(uint32_t* p, const F& v) {
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
  for (int k = 0; k < (int)(sizeof(F) / 4); k++) p[k] = s[k];
}

// ---- F_q / F_r: op 0 add 1 sub 2 mul 3 inverse 4 neg 5 sqr 6 inverse_vartime ----------------------------------------
// out: 9 words per element, the standard-form result and 1 if the op left a Montgomery representative >= p (which the
// conversion out of Montgomery form would hide)
template <class F>
__global__ void k_fp_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F x = ld<F>(a + 8 * i).to_mont(), y = ld<F>(b + 8 * i).to_mont(), r;
  switch (op) {
    case 0: r = x + y; break;
    case 1: r = x - y; break;
    case 2: r = x * y; break;
    case 3: r = x.inverse(); break;
    case 5: r = x.sqr(); break;
    case 6: r = x.inverse_vartime(); break;
    default: r = x.neg(); break;
  }
  st(out + 9 * i, r.from_mont());
  out[9 * i + 8] = r.geq_modulus();
}
template <class F>
__global__ void k_geq(const uint32_t* a, int* out, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = ld<F>(a + 8 * i).geq_modulus() ? 1 : 0;
}
template <class F>
__global__ void k_mul_full(const uint32_t* a, const uint32_t* b, uint32_t* w, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t x[8], y[8], r[16];
#pragma unroll
  for (int k = 0; k < 8; k++) {
    x[k] = a[8 * i + k];
    y[k] = b[8 * i + k];
  }
  F::mul_full(r, x, y);
#pragma unroll
  for (int k = 0; k < 16; k++) w[16 * i + k] = r[k];
}
template <class F>
__global__ void k_redc_wide(const uint32_t* t, uint32_t* out, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t x[16];
#pragma unroll
  for (int k = 0; k < 16; k++) x[k] = t[16 * i + k];
  st(out + 8 * i, F::redc_wide(x));
}

// ---- F_q^2: op 0 add 1 sub 2 mul 3 inverse 4 sqr 5 neg 6 inverse_vartime --------------------------------------------
// out: 17 words per element, the standard-form result and the flag of k_fp_op
template <class F2T>
__global__ void k_fq2_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F2T x = ld<F2T>(a + 16 * i).to_mont(), y = ld<F2T>(b + 16 * i).to_mont(), r;
  switch (op) {
    case 0: r = x + y; break;
    case 1: r = x - y; break;
    case 2: r = x * y; break;
    case 3: r = x.inverse(); break;
    case 4: r = x.sqr(); break;
    case 6: r = x.inverse_vartime(); break;
    default: r = x.neg(); break;
  }
  st(out + 17 * i, r.from_mont());
  out[17 * i + 16] = r.geq_modulus();
}

// ---- XYZZ: a = XYZZ (4 F), b = affine (first 2 F, op 0) or XYZZ (4 F, op 1); out = affine (2 F) ----------------------
// op 0 madd, 1 add, 2 dbl, 3 Jacobian round trip, 4 none (affine conversion by the vartime inversion)
template <class F>
__global__ void k_xyzz(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  constexpr int W = sizeof(F) / 4;
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  a += 4 * W * i;
  b += 4 * W * i;
  XYZZ<F> A{ld<F>(a).to_mont(), ld<F>(a + W).to_mont(), ld<F>(a + 2 * W).to_mont(), ld<F>(a + 3 * W).to_mont()};
  if (op == 0) {
    xyzz_madd(A, Affine<F>{ld<F>(b).to_mont(), ld<F>(b + W).to_mont()});
  } else if (op == 1) {
    xyzz_add(A, XYZZ<F>{ld<F>(b).to_mont(), ld<F>(b + W).to_mont(), ld<F>(b + 2 * W).to_mont(), ld<F>(b + 3 * W).to_mont()});
  } else if (op == 2) {
    A = xyzz_dbl(A);
  } else if (op == 3) {
    A = jacobian_to_xyzz(xyzz_to_jacobian(A));
  }
  Affine<F> r = op == 4 ? xyzz_to_affine<F, true>(A) : xyzz_to_affine(A);
  st(out + 2 * W * i, r.x.from_mont());
  st(out + 2 * W * i + W, r.y.from_mont());
}
// ---- the reference's Jacobian formulas: op 0 jac_add_ref(a, b), 1 jac_double_ref(a); X, Y, Z out ---------------------
template <class F>
__global__ void k_jac(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  constexpr int W = sizeof(F) / 4;
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  a += 3 * W * i;
  b += 3 * W * i;
  Jacobian<F> A{ld<F>(a).to_mont(), ld<F>(a + W).to_mont(), ld<F>(a + 2 * W).to_mont()};
  Jacobian<F> B{ld<F>(b).to_mont(), ld<F>(b + W).to_mont(), ld<F>(b + 2 * W).to_mont()};
  Jacobian<F> r = op == 0 ? jac_add_ref(A, B) : jac_double_ref(A);
  out += 3 * W * i;
  st(out, r.X.from_mont());
  st(out + W, r.Y.from_mont());
  st(out + 2 * W, r.Z.from_mont());
}

// ---- F_q^12, 96 words per element in the reference's [2][3][2] order (= the tower order of F12) -------------------
__device__ F12 ld12(const uint32_t* p) {
  F12 x;
  F2* xs[6] = {&x.a.a, &x.a.b, &x.a.c, &x.b.a, &x.b.b, &x.b.c};
  for (int k = 0; k < 6; k++) *xs[k] = ld<F2>(p + 16 * k).to_mont();
  return x;
}
__device__ void st12(uint32_t* p, const F12& x) {
  const F2* xs[6] = {&x.a.a, &x.a.b, &x.a.c, &x.b.a, &x.b.b, &x.b.c};
  for (int k = 0; k < 6; k++) st(p + 16 * k, xs[k]->from_mont());
}
// one thread per element: op 0 inverse, 1..3 Frobenius^op, 4 x^u (as t_f12_op), 5 f12_mul(a, b), 6 f12_sqr(a)
__global__ void k_f12_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F12 x = ld12(a + 96 * i), r;
  switch (op) {
    case 0: r = f12_inverse(x); break;
    case 1: r = f12_frobenius<1>(x); break;
    case 2: r = f12_frobenius<2>(x); break;
    case 3: r = f12_frobenius<3>(x); break;
    case 4: r = f12_exp_u(x); break;
    case 5: r = f12_mul(x, ld12(b + 96 * i)); break;
    default: r = f12_sqr(x); break;
  }
  st12(out + 96 * i, r);
}
// one warp per element, operands in registers r[0] = a, r[1] = b of the shared workspace:
//   op 0 r[2] = r[0] r[1]   1 r[0] = r[0] r[1]   2 r[1] = r[0] r[1]   3 r[0] = r[0] r[0]      (wp::f12_mul alias patterns)
//   op 4 inverse, 5..7 Frobenius^(op - 4), 8 x^u, 9 conjugate: r[2] from r[0]
__global__ void __launch_bounds__(32) k_f12_warp(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  __shared__ wp::Ws ws;
  const uint32_t lane = threadIdx.x;
  const size_t i = blockIdx.x;
  if (lane < 6) {
    ws.r[0][lane] = ld<F2>(a + 96 * i + 16 * lane).to_mont();
    ws.r[1][lane] = ld<F2>(b + 96 * i + 16 * lane).to_mont();
  }
  wp::wsync();
  wp::pairing_constants(ws);
  int d = 2;
  switch (op) {
    case 0: wp::f12_mul(ws, 2, 0, 1); break;
    case 1: wp::f12_mul(ws, 0, 0, 1); d = 0; break;
    case 2: wp::f12_mul(ws, 1, 0, 1); d = 1; break;
    case 3: wp::f12_sqr(ws, 0, 0); d = 0; break;
    case 4: wp::f12_inverse(ws, 2, 0); break;
    case 5: case 6: case 7: wp::f12_frobenius(ws, 2, 0, op - 4); break;
    case 8: wp::f12_exp_u(ws, 2, 0); break;
    default: wp::f12_conj(ws, 2, 0); break;
  }
  if (lane < 6) st(out + 96 * i + 16 * lane, ws.r[d][lane].from_mont());
}

// ---- GLV: k * P by one half-warp per product; P Jacobian (3 Fq), out Jacobian (3 Fq) --------------------------------
__global__ void __launch_bounds__(32) k_glv(const uint32_t* pts, const GlvScalars* g, uint32_t* out, size_t n) {
  const uint32_t t = threadIdx.x, grp = t >> 4;
  const size_t i = 2 * (size_t)blockIdx.x + grp;
  const size_t j = i < n ? i : n - 1;  // every lane takes part in the shuffles
  Jacobian<Fq> p{ld<Fq>(pts + 24 * j).to_mont(), ld<Fq>(pts + 24 * j + 8).to_mont(), ld<Fq>(pts + 24 * j + 16).to_mont()};
  Jacobian<Fq> r = glv_mul_halfwarp(p, g[j / 2].k[j & 1], g[j / 2].neg[j & 1], t);
  if ((t & 15u) == 0 && i < n) {
    st(out + 24 * i, r.X.from_mont());
    st(out + 24 * i + 8, r.Y.from_mont());
    st(out + 24 * i + 16, r.Z.from_mont());
  }
}

// ---- pairings of affine inputs: g1 = (x, y), g2 = (x.c0, x.c1, y.c0, y.c1); out 96 words -----------------------------
__global__ void k_pairing(int fast, const uint32_t* g1, const uint32_t* g2, uint32_t* out, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F2::B px = ld<F2::B>(g1 + 16 * i).to_mont(), py = ld<F2::B>(g1 + 16 * i + 8).to_mont();
  F2 qx = ld<F2>(g2 + 32 * i).to_mont(), qy = ld<F2>(g2 + 32 * i + 16).to_mont();
  st12(out + 96 * i, pairing_affine(px, py, qx, qy, fast != 0));
}
__global__ void __launch_bounds__(32) k_pairing_warp(const uint32_t* g1, const uint32_t* g2, uint32_t* out) {
  __shared__ wp::Ws ws;
  const size_t i = blockIdx.x;
  F2::B px = ld<F2::B>(g1 + 16 * i).to_mont(), py = ld<F2::B>(g1 + 16 * i + 8).to_mont();
  F2 qx = ld<F2>(g2 + 32 * i).to_mont(), qy = ld<F2>(g2 + 32 * i + 16).to_mont();
  wp::pairing(ws, px, py, qx, qy);
  if (threadIdx.x < 6) st(out + 96 * i + 16 * threadIdx.x, ws.r[wp::RF][threadIdx.x].from_mont());
}

// one launch over n elements of `in_words` words per operand (a and b) and `out_words` words of output
template <class Launch>
int run(size_t n, size_t in_words, const uint32_t* a, const uint32_t* b, size_t out_words, uint32_t* out, Launch launch) {
  if (n == 0) return 0;
  DevBuf da, db, dout;
  TRY(upload(da, a, n * in_words * 4));
  TRY(upload(db, b ? b : a, n * in_words * 4));
  TRY(upload(dout, nullptr, n * out_words * 4));
  launch(da.as<uint32_t>(), db.as<uint32_t>(), dout.as<uint32_t>());
  return finish(out, dout, n * out_words * 4);
}

}  // namespace

extern "C" {
// field: 0 F_q, 1 F_r ; inl: 0 the outlined (__noinline__) products, 1 the force-inlined ones (FqH / FrH) ; out 9 words each
int g_fp_op(int field, int inl, int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  return run(n, 8, a, b, 9, out, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    const unsigned g = blocks(n, 128);
    if (field == 0 && !inl) k_fp_op<Fq><<<g, 128>>>(op, x, y, o, n);
    else if (field == 0) k_fp_op<FqH><<<g, 128>>>(op, x, y, o, n);
    else if (!inl) k_fp_op<Fr><<<g, 128>>>(op, x, y, o, n);
    else k_fp_op<FrH><<<g, 128>>>(op, x, y, o, n);
  });
}
int g_geq(int field, int inl, const uint32_t* a, int* out, size_t n) {
  return run(n, 8, a, nullptr, 1, reinterpret_cast<uint32_t*>(out), [&](const uint32_t* x, const uint32_t*, uint32_t* o) {
    int* r = reinterpret_cast<int*>(o);
    const unsigned g = blocks(n, 128);
    if (field == 0 && !inl) k_geq<Fq><<<g, 128>>>(x, r, n);
    else if (field == 0) k_geq<FqH><<<g, 128>>>(x, r, n);
    else if (!inl) k_geq<Fr><<<g, 128>>>(x, r, n);
    else k_geq<FrH><<<g, 128>>>(x, r, n);
  });
}
// w = a * b as plain 512-bit integers (any 256-bit operands)
int g_mul_full(int inl, const uint32_t* a, const uint32_t* b, uint32_t* w, size_t n) {
  return run(n, 8, a, b, 16, w, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    if (inl) k_mul_full<FqH><<<blocks(n, 128), 128>>>(x, y, o, n);
    else k_mul_full<Fq><<<blocks(n, 128), 128>>>(x, y, o, n);
  });
}
// t / 2^256 mod p for 512-bit t < p * 2^256
int g_redc_wide(int field, int inl, const uint32_t* t, uint32_t* out, size_t n) {
  return run(n, 16, t, nullptr, 8, out, [&](const uint32_t* x, const uint32_t*, uint32_t* o) {
    const unsigned g = blocks(n, 128);
    if (field == 0 && !inl) k_redc_wide<Fq><<<g, 128>>>(x, o, n);
    else if (field == 0) k_redc_wide<FqH><<<g, 128>>>(x, o, n);
    else if (!inl) k_redc_wide<Fr><<<g, 128>>>(x, o, n);
    else k_redc_wide<FrH><<<g, 128>>>(x, o, n);
  });
}
// out 17 words each (k_fq2_op)
int g_fq2_op(int inl, int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  return run(n, 16, a, b, 17, out, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    if (inl) k_fq2_op<Fq2H><<<blocks(n, 128), 128>>>(op, x, y, o, n);
    else k_fq2_op<Fq2><<<blocks(n, 128), 128>>>(op, x, y, o, n);
  });
}
int g_g1_xyzz(int inl, int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  return run(n, 32, a, b, 16, out, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    if (inl) k_xyzz<FqH><<<blocks(n, 128), 128>>>(op, x, y, o, n);
    else k_xyzz<Fq><<<blocks(n, 128), 128>>>(op, x, y, o, n);
  });
}
int g_g2_xyzz(int inl, int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  return run(n, 64, a, b, 32, out, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    if (inl) k_xyzz<Fq2H><<<blocks(n, 128), 128>>>(op, x, y, o, n);
    else k_xyzz<Fq2><<<blocks(n, 128), 128>>>(op, x, y, o, n);
  });
}
int g_g1_jac(int inl, int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  return run(n, 24, a, b, 24, out, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    if (inl) k_jac<FqH><<<blocks(n, 128), 128>>>(op, x, y, o, n);
    else k_jac<Fq><<<blocks(n, 128), 128>>>(op, x, y, o, n);
  });
}
int g_g2_jac(int inl, int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  return run(n, 48, a, b, 48, out, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    if (inl) k_jac<Fq2H><<<blocks(n, 128), 128>>>(op, x, y, o, n);
    else k_jac<Fq2><<<blocks(n, 128), 128>>>(op, x, y, o, n);
  });
}
int g_f12_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  return run(n, 96, a, b, 96, out, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    k_f12_op<<<blocks(n, 64), 64>>>(op, x, y, o, n);
  });
}
int g_f12_warp(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
  return run(n, 96, a, b, 96, out, [&](const uint32_t* x, const uint32_t* y, uint32_t* o) {
    k_f12_warp<<<(unsigned)n, 32>>>(op, x, y, o);
  });
}
// k * P: pts n Jacobian points (24 words), ks n standard-form scalars (8 words) split by glv_decompose; out Jacobian.
// Returns -1 if a decomposition fails.
int g_glv_mul(const uint32_t* pts, const uint32_t* ks, uint32_t* out, size_t n) {
  if (n == 0) return 0;
  std::vector<GlvScalars> g((n + 1) / 2);
  std::memset(g.data(), 0, g.size() * sizeof(GlvScalars));
  for (size_t i = 0; i < n; i++) {
    Fr k;
    std::memcpy(&k, ks + 8 * i, sizeof(Fr));
    if (glv_decompose(k, g[i / 2].k[i & 1], g[i / 2].neg[i & 1])) return -1;
  }
  DevBuf dg;
  TRY(upload(dg, g.data(), g.size() * sizeof(GlvScalars)));
  return run(n, 24, pts, nullptr, 24, out, [&](const uint32_t* x, const uint32_t*, uint32_t* o) {
    k_glv<<<(unsigned)((n + 1) / 2), 32>>>(x, dg.as<GlvScalars>(), o, n);
  });
}
// mode 0: pairing_affine, plain final exponentiation; 1: fast final exponentiation; 2: wp::pairing (one warp each)
int g_pairing(int mode, const uint32_t* g1, const uint32_t* g2, uint32_t* out, size_t n) {
  if (n == 0) return 0;
  DevBuf d1, d2, dout;
  TRY(upload(d1, g1, n * 64));
  TRY(upload(d2, g2, n * 128));
  TRY(upload(dout, nullptr, n * 384));
  if (mode == 2) k_pairing_warp<<<(unsigned)n, 32>>>(d1.as<uint32_t>(), d2.as<uint32_t>(), dout.as<uint32_t>());
  else k_pairing<<<blocks(n, 32), 32>>>(mode, d1.as<uint32_t>(), d2.as<uint32_t>(), dout.as<uint32_t>(), n);
  return finish(out, dout, n * 384);
}
}
