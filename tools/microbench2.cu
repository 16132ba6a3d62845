// microbench2.cu -- exact-instruction integer pipe probes for sm_90a (inline PTX so the compiler cannot re-associate):
// is IMAD.HI (a right shift on the FMA pipe) full rate?  how do the delta-swap formulations compare?  Diagnostic only.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define ITERS 2048
__device__ __forceinline__ uint32_t lop3_sel(uint32_t a, uint32_t b, uint32_t m) {  // (a & m) | (b & ~m)
  uint32_t d;
  asm volatile("lop3.b32 %0, %1, %2, %3, 0xE4;" : "=r"(d) : "r"(a), "r"(b), "r"(m));
  return d;
}
__device__ __forceinline__ uint32_t mulhi(uint32_t a, uint32_t b) {
  uint32_t d;
  asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
__device__ __forceinline__ uint32_t madhi(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm volatile("mad.hi.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ uint32_t mullo(uint32_t a, uint32_t b) {
  uint32_t d;
  asm volatile("mul.lo.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
__device__ __forceinline__ uint32_t shr(uint32_t a, uint32_t n) {
  uint32_t d;
  asm volatile("shr.b32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(n));
  return d;
}
__device__ __forceinline__ uint32_t bfind(uint32_t a) {
  uint32_t d;
  asm volatile("bfind.u32 %0, %1;" : "=r"(d) : "r"(a));
  return d;
}

template <int OP>
__global__ void k(uint32_t *out, unsigned long long *cycles, uint32_t seed) {
  uint32_t a[8];
#pragma unroll
  for (int i = 0; i < 8; i++) a[i] = seed * (threadIdx.x + 1) + i * 0x9E3779B9u;
  const uint32_t m = 0x0F0F0F0Fu ^ (seed & 1u), c16 = 16u + (seed & 2u), c28 = 0x10000000u + (seed & 4u), s4 = 4u + (seed & 8u);
  unsigned long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
      uint32_t lo = a[i], hi = a[i + 1];
      if (OP == 0) { a[i] = lop3_sel(lo, hi, m); a[i + 1] = lop3_sel(hi, lo, m); }                   // 2 LOP3
      if (OP == 1) { a[i] = mulhi(lo, c28) ^ hi; a[i + 1] = mulhi(hi, c28) ^ lo; }                    // 2 IMAD.HI + 2 LOP3
      if (OP == 2) { a[i] = mulhi(lo, c28); a[i + 1] = mulhi(hi, c28) + 1; }                          // IMAD.HI (+ an add)
      if (OP == 3) { a[i] = lop3_sel(lo, mullo(hi, c16), m); a[i + 1] = lop3_sel(shr(lo, s4), hi, m); }   // dswap today: 2 LOP3 + IMAD + SHF
      if (OP == 4) { a[i] = lop3_sel(lo, mullo(hi, c16), m); a[i + 1] = lop3_sel(mulhi(lo, c28), hi, m); } // dswap proposed: 2 LOP3 + IMAD + IMAD.HI
      if (OP == 5) { a[i] = madhi(lo, c16, mullo(hi, c16)); a[i + 1] = madhi(hi, c16, mullo(lo, c16)); }  // funnel shift on the FMA pipe: IMAD + IMAD.HI
      if (OP == 6) { a[i] = bfind(lo) + hi; a[i + 1] = bfind(hi) + lo; }                               // FLO + IADD
      if (OP == 7) { a[i] = __funnelshift_l(lo, hi, s4); a[i + 1] = __funnelshift_l(hi, lo, s4); }     // SHF
    }
  }
  unsigned long long t1 = clock64();
  uint32_t r = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) r ^= a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = r;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int OP>
void run(const char *name, int warp_instr_per_pair, int warps_per_sm) {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  int threads = 32 * warps_per_sm;
  uint32_t *out;
  unsigned long long *cyc;
  cudaMalloc(&out, sizeof(uint32_t) * sms * threads);
  cudaMalloc(&cyc, sizeof(unsigned long long) * sms);
  k<OP><<<sms, threads>>>(out, cyc, 12345);
  k<OP><<<sms, threads>>>(out, cyc, 12345);
  cudaDeviceSynchronize();
  unsigned long long h[256];
  cudaMemcpy(h, cyc, sizeof(unsigned long long) * sms, cudaMemcpyDeviceToHost);
  double avg = 0;
  for (int i = 0; i < sms; i++) avg += double(h[i]);
  avg /= sms;
  const double pairs = double(ITERS) * 4 * warps_per_sm;  // warp-level pair bodies per SM
  printf("%-52s warps/SM=%2d  cycles per pair body per SMSP = %6.2f  (%d warp-instr each)\n", name, warps_per_sm, avg / (pairs / 4.0),
         warp_instr_per_pair);
  cudaFree(out); cudaFree(cyc);
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  printf("%s, %d SMs\n", p.name, p.multiProcessorCount);
  for (int w : {16, 32}) {
    run<0>("2 LOP3", 2, w);
    run<7>("2 SHF", 2, w);
    run<2>("2 IMAD.HI (+1 add)", 3, w);
    run<1>("2 IMAD.HI + 2 LOP3", 4, w);
    run<3>("dswap: 2 LOP3 + IMAD.SHL + SHF.R", 4, w);
    run<4>("dswap: 2 LOP3 + IMAD.SHL + IMAD.HI", 4, w);
    run<5>("2 x (IMAD + IMAD.HI) funnel on FMA pipe", 4, w);
    run<6>("2 x (FLO + IADD)", 4, w);
  }
  return 0;
}
