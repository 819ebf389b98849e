// Microbenchmark (development aid; nvcc -gencode arch=compute_90a,code=sm_90a -O3): do the integer-multiply pipe (IMAD.WIDE.X carry chains — what the
// Montgomery kernels are made of) and the FP64 pipe (DFMA, the Emmart-style 52-bit-limb route) + the ALU pipe (64-bit
// integer adds of the DFMA results) run CONCURRENTLY when different warps of an SM execute them?
//   mode 0: every warp runs the IMAD.WIDE.X chain        mode 1: every warp runs DFMA(+DADD) + int64 adds
//   mode 2: even warps IMAD, odd warps DFMA              mode 3: DFMA only (no integer adds)      mode 4: DADD only
//   mode 5: plain IMAD.WIDE.U32 (64-bit addend, no carry flags), loop-variant operands
// Operands vary per iteration (the chain's own outputs feed back) so ptxas cannot hoist the products.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

// SM count and peak SM clock of device 0 (the rates below are per SM and per clock at that peak clock).
static int dev_sms() { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, 0); return v; }
static double dev_clk_hz() { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrClockRate, 0); return v * 1e3; }

__device__ __forceinline__ void imad_chain(uint32_t (&r)[8], uint32_t a, uint32_t& b) {
  asm volatile(
      "mad.lo.cc.u32 %0, %8, %9, %0; madc.hi.cc.u32 %1, %8, %9, %1; madc.lo.cc.u32 %2, %8, %9, %2; madc.hi.cc.u32 %3, %8, %9, %3;"
      "madc.lo.cc.u32 %4, %8, %9, %4; madc.hi.cc.u32 %5, %8, %9, %5; madc.lo.cc.u32 %6, %8, %9, %6; madc.hi.u32 %7, %8, %9, %7;"
      : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "+r"(r[3]), "+r"(r[4]), "+r"(r[5]), "+r"(r[6]), "+r"(r[7]) : "r"(a), "r"(b));
}

__global__ void __launch_bounds__(512) k(uint32_t* out, uint32_t a0, double d0, int iters, int mode) {
  const int warp = threadIdx.x >> 5;
  int path = mode == 2 ? (warp & 1) : (mode == 0 ? 0 : mode);
  uint32_t acc = 0;
  if (path == 0) {
    uint32_t r[8] = {1, 2, 3, 4, 5, 6, 7, 8}, s[8] = {8, 7, 6, 5, 4, 3, 2, 1};
    uint32_t a = a0 + threadIdx.x, b = a0 * 3 + blockIdx.x;
    for (int i = 0; i < iters; i++) {
      // two independent 4-pair chains per iteration; operands come from the other chain's result
      imad_chain(r, a, b);
      imad_chain(s, b, a);
      a ^= s[1];
      b += r[2];
    }
    for (int i = 0; i < 8; i++) acc ^= r[i] ^ s[i];
  } else if (path == 1) {
    // 8 products per iteration, each: hi = fma.rz(a,b,C1); t = C2 - hi; lo = fma.rz(a,b,t); two int64 adds of the bit patterns
    double a = d0 + threadIdx.x, b = d0 * 3.0 + blockIdx.x;
    const double C1 = 20282409603651670423947251286016.0;   // 2^104
    const double C2 = C1 + 4503599627370496.0;              // 2^104 + 2^52
    long long h0 = 0, h1 = 0, h2 = 0, h3 = 0, l0 = 0, l1 = 0, l2 = 0, l3 = 0;
    for (int i = 0; i < iters; i++) {
#define PROD(H, L, x, y)                                          \
  {                                                               \
    double hi = __fma_rz(x, y, C1);                               \
    double t = C2 - hi;                                           \
    double lo = __fma_rz(x, y, t);                                \
    H += __double_as_longlong(hi);                                \
    L += __double_as_longlong(lo);                                \
  }
      PROD(h0, l0, a, b) PROD(h1, l1, a + 1.0, b) PROD(h2, l2, a, b + 1.0) PROD(h3, l3, a + 2.0, b)
      PROD(h0, l1, b, b) PROD(h1, l2, a, a) PROD(h2, l3, a + 3.0, b) PROD(h3, l0, a, b + 3.0)
      a = (double)(int)(l0 & 0xfffff) + 1.0;   // loop-variant operands (2 conversions per 8 products)
      b += 1.0;
    }
    acc = (uint32_t)(h0 ^ h1 ^ h2 ^ h3 ^ l0 ^ l1 ^ l2 ^ l3) ^ (uint32_t)((h0 ^ l3) >> 32);
  } else if (path == 3) {
    double a = d0 + threadIdx.x, b = d0 * 3.0 + blockIdx.x;
    double x0 = 1, x1 = 2, x2 = 3, x3 = 4, x4 = 5, x5 = 6, x6 = 7, x7 = 8;
    for (int i = 0; i < iters; i++) {
      x0 = __fma_rz(a, b, x0); x1 = __fma_rz(a, x0, x1); x2 = __fma_rz(b, x1, x2); x3 = __fma_rz(a, x2, x3);
      x4 = __fma_rz(a, b, x4); x5 = __fma_rz(a, x4, x5); x6 = __fma_rz(b, x5, x6); x7 = __fma_rz(a, x6, x7);
      a = x3 * 1e-300; b = x7 * 1e-300;   // keep magnitudes bounded (2 DMUL per 8 DFMA)
    }
    acc = (uint32_t)__double_as_longlong(x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7);
  } else if (path == 4) {
    double a = d0 + threadIdx.x;
    double x0 = 1, x1 = 2, x2 = 3, x3 = 4, x4 = 5, x5 = 6, x6 = 7, x7 = 8;
    for (int i = 0; i < iters; i++) {
      x0 += a; x1 += x0; x2 += x1; x3 += x2; x4 += a; x5 += x4; x6 += x5; x7 += x6;
      a = x3 - x7;
    }
    acc = (uint32_t)__double_as_longlong(x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7);
  } else if (path == 5) {
    uint64_t w0 = 1, w1 = 2, w2 = 3, w3 = 4, w4 = 5, w5 = 6, w6 = 7, w7 = 8;
    uint32_t a = a0 + threadIdx.x, b = a0 * 3 + blockIdx.x;
    for (int i = 0; i < iters; i++) {
#define W(x, p, q) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(x) : "r"(p), "r"(q));
      // eight DISTINCT products (identical ones would be merged by ptxas)
      const uint32_t c = a ^ 0x9e3779b9u, d = b + 0x7f4a7c15u, e = a + b;
      W(w0, a, b) W(w1, a, c) W(w2, b, c) W(w3, a, d) W(w4, b, d) W(w5, c, d) W(w6, a, e) W(w7, b, e)
      a += (uint32_t)w3; b ^= (uint32_t)(w7 >> 32);
    }
    acc = (uint32_t)(w0 ^ w1 ^ w2 ^ w3 ^ w4 ^ w5 ^ w6 ^ w7) ^ (uint32_t)((w0 ^ w5) >> 32);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

float run(int mode, int iters, uint32_t* d) {
  int blocks = dev_sms() * 4, threads = 512;
  k<<<blocks, threads>>>(d, 3, 5.0, 64, mode);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  k<<<blocks, threads>>>(d, 3, 5.0, iters, mode);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  return ms;
}

int main() {
  uint32_t* d;
  cudaMalloc(&d, dev_sms() * 4 * 512 * 4);
  const int iters = 20000;
  const double sms = dev_sms(), warps = sms * 4 * 16, clk = dev_clk_hz();
  float t0 = run(0, iters, d), t1 = run(1, iters, d), t2 = run(2, iters, d), t3 = run(3, iters, d), t4 = run(4, iters, d), t5 = run(5, iters, d);
  // per-SMSP cycles per warp-instruction group
  auto cyc = [&](float ms, double warp_ops) { return ms * 1e-3 * clk * sms * 4 / warp_ops; };
  printf("mode 0 IMAD.WIDE.X chains      %8.3f ms   %.2f SMSP-cycles per wide MAC warp-instr (8 per iteration)\n", t0, cyc(t0, warps * iters * 8));
  printf("mode 5 IMAD.WIDE (no carry)    %8.3f ms   %.2f SMSP-cycles per wide MAC warp-instr (8 per iteration)\n", t5, cyc(t5, warps * iters * 8));
  printf("mode 3 DFMA only               %8.3f ms   %.2f SMSP-cycles per DFMA warp-instr (8 + 2 DMUL per iteration)\n", t3, cyc(t3, warps * iters * 10));
  printf("mode 4 DADD only               %8.3f ms   %.2f SMSP-cycles per DADD warp-instr (9 per iteration)\n", t4, cyc(t4, warps * iters * 9));
  printf("mode 1 DFMA products + int64   %8.3f ms   %.2f SMSP-cycles per 52x52 product (2 DFMA + DADD + 2 int64 adds)\n", t1, cyc(t1, warps * iters * 8));
  printf("mode 2 even warps 0, odd 1     %8.3f ms   additive pipes would give %.3f ms, one shared pipe %.3f ms\n", t2,
         (t0 > t1 ? t0 : t1) / 2, (t0 + t1) / 2);
  // Montgomery multiply equivalents: IMAD route 136 wide MACs; DFMA route ~55 products of 52x52 bits
  printf("=> 254-bit Montgomery multiply, per SMSP: IMAD route %.0f cycles (136 wide MACs), DFMA route %.0f cycles (55 products)\n",
         136 * cyc(t0, warps * iters * 8), 55 * cyc(t1, warps * iters * 8));
  return 0;
}
