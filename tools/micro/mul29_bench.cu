// Microbenchmark (development aid): throughput of the two Montgomery multiplications of fp.cuh —
// mul_impl (8 x 32-bit limbs, IMAD.WIDE.U32.X carry chains) against mul29_impl (nine 29-bit limbs, carry-free IMAD.WIDE.U32) —
// as out-of-line device functions called from a dependent chain per thread (the shape of the bucket kernels' inner loops),
// at several occupancies, plus a bit-for-bit comparison of the two on random operands.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "fp.cuh"
using namespace b200;

// SM count and peak SM clock of device 0 (the rates below are per SM and per clock at that peak clock).
static int dev_sms() { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, 0); return v; }
static double dev_clk_hz() { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrClockRate, 0); return v * 1e3; }

// ---- the experiment: carry-free Montgomery multiplication on nine 29-bit limbs (same result as Fq::mul_impl) -------------
// A 64-bit column accumulator holds 18 products of 29-bit limbs without overflowing, so no partial product needs a carry
// flag.  The reduction takes eight 29-bit digits and one 24-bit digit (232 + 24 = 256: R stays 2^256); the quotient columns then
// sit at bit offsets 5 + 29 k and are packed straight into 32-bit words.  ptxas splits every mad.wide.u32 with a 64-bit
// addend into IMAD.WIDE.U32 (RZ addend) + a 3-input IADD3 / IADD3.X pair, and 81 + 81 products replace 64 + 64.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I go-snark-study_b200/csrc -o tools/micro/mul29_bench tools/micro/mul29_bench.cu
__device__ __constant__ uint32_t kQ29[9] = {0x187cfd47u, 0x010460b6u, 0x1c72a34fu, 0x02d522d0u, 0x1585d978u, 0x02db40c0u, 0x00a6e141u, 0x0e5c2634u, 0x0030644eu};
__device__ __forceinline__ uint64_t mad_wide64(uint32_t a, uint32_t b, uint64_t c) {
  uint64_t r;
  asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(r) : "r"(a), "r"(b), "l"(c));
  return r;
}
__device__ __forceinline__ void unpack29(const uint32_t* w, uint32_t* l) {
#pragma unroll
  for (int k = 0; k < 9; k++) {
    const int bit = 29 * k, wi = bit >> 5, sh = bit & 31;
    uint32_t v = w[wi] >> sh;
    if (sh > 3 && wi + 1 < 8) v |= w[wi + 1] << (32 - sh);
    l[k] = v & 0x1fffffffu;
  }
}
__device__ __forceinline__ Fq mul29(const Fq& a, const Fq& b) {
  constexpr uint32_t M29 = 0x1fffffffu, INV29 = FqParams::INV & M29;
  uint32_t al[9], bl[9];
  unpack29(a.l, al);
  unpack29(b.l, bl);
  uint64_t acc[17];
#pragma unroll
  for (int k = 0; k < 17; k++) acc[k] = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {
#pragma unroll
    for (int j = 0; j < 9; j++) acc[i + j] = mad_wide64(al[i], bl[j], acc[i + j]);
    const uint32_t q = ((uint32_t)acc[i] * INV29) & (i < 8 ? M29 : 0x00ffffffu);
#pragma unroll
    for (int j = 0; j < 9; j++) acc[i + j] = mad_wide64(q, kQ29[j], acc[i + j]);
    if (i < 8) acc[i + 1] += acc[i] >> 29;
  }
  // V = (acc[8] >> 24) + sum_k acc[9 + k] << (5 + 29 k)  <  2p
  uint32_t r[9];
  {
    uint64_t t = acc[8] >> 24;
    r[0] = (uint32_t)t;
    r[1] = (uint32_t)(t >> 32);
#pragma unroll
    for (int k = 2; k < 9; k++) r[k] = 0;
  }
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int off = 5 + 29 * k, m = off >> 5, s = off & 31;
    const uint32_t lo = (uint32_t)acc[9 + k], hi = (uint32_t)(acc[9 + k] >> 32);
    r[m] = cc::add_cc(r[m], lo << s);
    r[m + 1] = cc::addc_cc(r[m + 1], (lo >> (32 - s)) | (hi << s));
    r[m + 2] = cc::addc(r[m + 2], hi >> (32 - s));
  }
  Fq o;
#pragma unroll
  for (int k = 0; k < 8; k++) o.l[k] = r[k];
  Fq::final_sub(o.l);
  return o;
}

template <int V> __device__ __noinline__ Fq mul_v(Fq a, Fq b) { return V == 0 ? Fq::mul_impl(a, b) : mul29(a, b); }

template <int V>
__global__ void __launch_bounds__(128) k_chain(Fq* io, int iters) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  Fq x = io[2 * t], y = io[2 * t + 1], z = x + y;
  for (int i = 0; i < iters; i++) {   // two independent chains, like the backward pass's inv_run and lambda products
    x = mul_v<V>(x, y);
    z = mul_v<V>(z, x);
  }
  io[2 * t] = x;
  io[2 * t + 1] = z;
}
__global__ void k_cmp(const Fq* in, int n, int* bad) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  Fq a = in[2 * t], b = in[2 * t + 1];
  for (int i = 0; i < 64; i++) {
    Fq u = Fq::mul_impl(a, b), v = mul29(a, b);
    if (!(u == v)) atomicAdd(bad, 1);
    a = b;
    b = u;
  }
}

int main() {
  const int max_threads = dev_sms() * 16 * 128;
  Fq* d;
  cudaMalloc(&d, sizeof(Fq) * 2 * max_threads);
  // operands: arbitrary reduced values (top limb small)
  uint32_t* h = (uint32_t*)malloc(sizeof(Fq) * 2 * max_threads);
  uint64_t s = 88172645463325252ull;
  for (size_t i = 0; i < (size_t)max_threads * 16; i++) {
    s ^= s << 13; s ^= s >> 7; s ^= s << 17;
    h[i] = (uint32_t)s;
    if ((i & 7) == 7) h[i] &= 0x0fffffffu;
  }
  cudaMemcpy(d, h, sizeof(Fq) * 2 * max_threads, cudaMemcpyHostToDevice);
  int* bad;
  cudaMalloc(&bad, 4);
  cudaMemset(bad, 0, 4);
  k_cmp<<<(max_threads + 127) / 128, 128>>>(d, max_threads, bad);
  int hb = -1;
  cudaMemcpy(&hb, bad, 4, cudaMemcpyDeviceToHost);
  printf("bit-for-bit comparison, %d x 64 products: %d mismatches (%s)\n", max_threads, hb, cudaGetErrorString(cudaGetLastError()));
  const int iters = 2000;
  for (int cta_per_sm : {2, 4, 5, 8, 12, 16}) {
    float ms[2];
    for (int v = 0; v < 2; v++) {
      int blocks = dev_sms() * cta_per_sm;
      cudaMemcpy(d, h, sizeof(Fq) * 2 * max_threads, cudaMemcpyHostToDevice);
      if (v == 0) k_chain<0><<<blocks, 128>>>(d, 10); else k_chain<1><<<blocks, 128>>>(d, 10);
      cudaEvent_t e0, e1;
      cudaEventCreate(&e0); cudaEventCreate(&e1);
      cudaEventRecord(e0);
      if (v == 0) k_chain<0><<<blocks, 128>>>(d, iters); else k_chain<1><<<blocks, 128>>>(d, iters);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      cudaEventElapsedTime(&ms[v], e0, e1);
    }
    double muls = (double)dev_sms() * cta_per_sm * 128 * iters * 2;
    auto cyc = [&](float m) { return m * 1e-3 * dev_clk_hz() * dev_sms() * 4 / (muls / 32); };   // SMSP-cycles per warp-level multiply
    printf("%2d CTAs/SM (%2d warps/SMSP): mul_impl %7.3f ms = %5.0f SMSP-cycles/warp-mul (%.1f Gmul/s)   mul29_impl %7.3f ms = %5.0f (%.1f Gmul/s)   x%.2f\n",
           cta_per_sm, cta_per_sm, ms[0], cyc(ms[0]), muls / ms[0] / 1e6, ms[1], cyc(ms[1]), muls / ms[1] / 1e6, ms[0] / ms[1]);
  }
  return 0;
}
