// microbench.cu -- integer pipe throughput on sm_90a (SURVEY.md section 7, hard part 1:
// "measure LOP3/PRMT/IADD3/IMAD throughput on the box before designing").
// Prints lane-ops per clock per SM for a few instruction mixes.  Diagnostic tool only.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define ITERS 4096
template <int OP>
__global__ void k(uint32_t *out, unsigned long long *cycles, uint32_t seed) {
  uint32_t a[8];
#pragma unroll
  for (int i = 0; i < 8; i++) a[i] = seed * (threadIdx.x + 1) + i * 0x9E3779B9u;
  uint32_t m = seed | 0x55555555u, s = (seed & 7) + 1;
  unsigned long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      if (OP == 0) a[i] = (a[i] & m) ^ (a[(i + 1) & 7] | ~m);             // LOP3
      if (OP == 1) a[i] = __funnelshift_l(a[i], a[(i + 1) & 7], s);       // SHF
      if (OP == 2) a[i] = __byte_perm(a[i], a[(i + 1) & 7], 0x5140 + s);  // PRMT
      if (OP == 3) a[i] = a[i] * 0x01020408u + a[(i + 1) & 7];            // IMAD
      if (OP == 4) a[i] = a[i] + a[(i + 1) & 7] + m;                      // IADD3
      if (OP == 5) {                                                       // LOP3 + IMAD mix 1:1
        a[i] = (a[i] & m) ^ (a[(i + 1) & 7] | ~m);
        a[(i + 3) & 7] = a[(i + 3) & 7] * 0x01020408u + a[i];
      }
      if (OP == 6) {                                                       // delta-swap shape: 2 shifts + 2 lop3
        uint32_t lo = a[i], hi = a[(i + 1) & 7];
        a[i] = (lo & m) | ((hi << 2) & ~m);
        a[(i + 1) & 7] = ((lo >> 2) & m) | (hi & ~m);
      }
      if (OP == 7) a[i] = __popc(a[i]) + a[(i + 1) & 7];                  // POPC
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
void run(const char *name, int ops_per_inner, int warps_per_sm) {
  int dev = 0, sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int threads = 32 * warps_per_sm;  // one block per SM
  uint32_t *out;
  unsigned long long *cyc;
  cudaMalloc(&out, sizeof(uint32_t) * sms * threads);
  cudaMalloc(&cyc, sizeof(unsigned long long) * sms);
  k<OP><<<sms, threads>>>(out, cyc, 12345);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  k<OP><<<sms, threads>>>(out, cyc, 12345);
  cudaEventRecord(e1);
  cudaDeviceSynchronize();
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  unsigned long long h[256];
  cudaMemcpy(h, cyc, sizeof(unsigned long long) * sms, cudaMemcpyDeviceToHost);
  double avg = 0;
  for (int i = 0; i < sms; i++) avg += double(h[i]);
  avg /= sms;
  double laneops = double(ITERS) * 8 * ops_per_inner * threads;
  printf("%-28s warps/SM=%2d  lane-ops/clk/SM = %7.1f   (%.3f ms, %.0f cycles)\n", name, warps_per_sm, laneops / avg, ms, avg);
  cudaFree(out); cudaFree(cyc);
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  printf("%s, %d SMs, clock %d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
  for (int w : {8, 16, 32}) {
    run<0>("LOP3", 1, w);
    run<1>("SHF (funnel)", 1, w);
    run<2>("PRMT", 1, w);
    run<3>("IMAD", 1, w);
    run<4>("IADD3", 1, w);
    run<5>("LOP3+IMAD 1:1", 2, w);
    run<6>("delta-swap (2 SHF + 2 LOP3)", 4, w);
    run<7>("POPC+IADD", 2, w);
  }
  return 0;
}
