// Microbenchmark: per-SM throughput of the integer multiply instructions the
// Montgomery kernels are built from.  Development aid:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/imad_bench tools/micro/imad_bench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

// SM count and peak SM clock of device 0 (the rates below are per SM and per clock at that peak clock).
static int dev_sms() { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, 0); return v; }
static double dev_clk_hz() { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrClockRate, 0); return v * 1e3; }

template <int MODE>
__global__ void k(uint32_t* out, uint32_t a0, uint32_t b0, int iters) {
  uint32_t a = a0 + threadIdx.x, b = b0 + blockIdx.x;
  uint32_t r0 = 1, r1 = 2, r2 = 3, r3 = 4, r4 = 5, r5 = 6, r6 = 7, r7 = 8;
  uint64_t w0 = 1, w1 = 2, w2 = 3, w3 = 4, w4 = 5, w5 = 6, w6 = 7, w7 = 8;
  for (int i = 0; i < iters; i++) {
    if (MODE == 0) {  // IMAD.WIDE.U32 independent
#define W(x) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(x) : "r"(a), "r"(b));
      W(w0) W(w1) W(w2) W(w3) W(w4) W(w5) W(w6) W(w7)
    } else if (MODE == 1) {  // IMAD lo
#define L(x) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(x) : "r"(a), "r"(b));
      L(r0) L(r1) L(r2) L(r3) L(r4) L(r5) L(r6) L(r7)
    } else if (MODE == 2) {  // IMAD.HI
#define H(x) asm volatile("mad.hi.u32 %0, %1, %2, %0;" : "+r"(x) : "r"(a), "r"(b));
      H(r0) H(r1) H(r2) H(r3) H(r4) H(r5) H(r6) H(r7)
    } else if (MODE == 3) {  // carry chain of wide mads: 4 pairs, two independent chains
      asm volatile(
          "mad.lo.cc.u32 %0, %8, %9, %0; madc.hi.cc.u32 %1, %8, %9, %1; madc.lo.cc.u32 %2, %8, %9, %2; madc.hi.cc.u32 %3, %8, %9, %3;"
          "madc.lo.cc.u32 %4, %8, %9, %4; madc.hi.cc.u32 %5, %8, %9, %5; madc.lo.cc.u32 %6, %8, %9, %6; madc.hi.u32 %7, %8, %9, %7;"
          : "+r"(r0), "+r"(r1), "+r"(r2), "+r"(r3), "+r"(r4), "+r"(r5), "+r"(r6), "+r"(r7) : "r"(a), "r"(b));
      uint32_t s0 = (uint32_t)w0, s1 = (uint32_t)w1, s2 = (uint32_t)w2, s3 = (uint32_t)w3, s4 = (uint32_t)w4, s5 = (uint32_t)w5, s6 = (uint32_t)w6, s7 = (uint32_t)w7;
      asm volatile(
          "mad.lo.cc.u32 %0, %8, %9, %0; madc.hi.cc.u32 %1, %8, %9, %1; madc.lo.cc.u32 %2, %8, %9, %2; madc.hi.cc.u32 %3, %8, %9, %3;"
          "madc.lo.cc.u32 %4, %8, %9, %4; madc.hi.cc.u32 %5, %8, %9, %5; madc.lo.cc.u32 %6, %8, %9, %6; madc.hi.u32 %7, %8, %9, %7;"
          : "+r"(s0), "+r"(s1), "+r"(s2), "+r"(s3), "+r"(s4), "+r"(s5), "+r"(s6), "+r"(s7) : "r"(b), "r"(a));
      w0 = s0; w1 = s1; w2 = s2; w3 = s3; w4 = s4; w5 = s5; w6 = s6; w7 = s7;
    } else if (MODE == 4) {  // IADD3
#define A(x) asm volatile("add.u32 %0, %0, %1;" : "+r"(x) : "r"(a));
      A(r0) A(r1) A(r2) A(r3) A(r4) A(r5) A(r6) A(r7)
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = r0 ^ r1 ^ r2 ^ r3 ^ r4 ^ r5 ^ r6 ^ r7 ^ (uint32_t)(w0 ^ w1 ^ w2 ^ w3 ^ w4 ^ w5 ^ w6 ^ w7) ^ (uint32_t)((w0 ^ w7) >> 32);
}

template <int MODE>
void run(const char* name, int ops_per_iter) {
  uint32_t* d;
  int blocks = dev_sms() * 4, threads = 512, iters = 20000;
  cudaMalloc(&d, blocks * threads * 4);
  k<MODE><<<blocks, threads>>>(d, 3, 5, 100);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  k<MODE><<<blocks, threads>>>(d, 3, 5, iters);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  double ops = (double)blocks * threads * iters * ops_per_iter;   // thread-level ops
  double per_sm_clk = ops / (ms * 1e-3) / dev_sms() / dev_clk_hz();
  printf("%-28s %8.3f ms  %7.2f Tops/s  %6.1f thread-ops/clk/SM (at %.0f MHz)\n", name, ms, ops / ms / 1e9, per_sm_clk, dev_clk_hz() / 1e6);
  cudaFree(d);
}

int main() {
  run<0>("IMAD.WIDE.U32 (indep)", 8);
  run<1>("IMAD.LO", 8);
  run<2>("IMAD.HI", 8);
  run<3>("mad.lo/hi.cc chain (pairs)", 8);   // counted as 8 WIDE-equivalents (16 half ops)
  run<4>("IADD", 8);
  return 0;
}
