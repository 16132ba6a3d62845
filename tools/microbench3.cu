// microbench3: what bounds a launch and the host-pointer path on this box (tuning aid, not the product)
//   1. event-to-event time of empty kernels: grid / block / dynamic shared memory / a 128-byte __grid_constant__ parameter
//   2. copy engine: pinned H2D, D2H, both at once; H2D from pageable memory
//   3. kernel stores to mapped host memory
//   4. memcpy pageable -> pinned with T threads
// build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/microbench3 tools/microbench3.cu -lpthread
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <thread>
#include <vector>

struct Big { uint64_t w[16]; };
__global__ void k_empty(uint32_t *p) { if (p && threadIdx.x == 0 && blockIdx.x == 0) *p = 1; }
__global__ void k_empty_big(const __grid_constant__ Big b, uint32_t *p) { if (p && threadIdx.x == 0 && blockIdx.x == 0) *p = uint32_t(b.w[3]); }
__global__ void k_smem(uint32_t *p) {
  extern __shared__ uint8_t sm[];
  if (threadIdx.x == 0) sm[0] = 1;
  __syncthreads();
  if (p && threadIdx.x == 0 && blockIdx.x == 0) *p = sm[0];
}
__global__ void k_store_host(uint4 *dst, size_t nvec) {
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += size_t(gridDim.x) * blockDim.x) dst[i] = make_uint4(uint32_t(i), 1, 2, 3);
}

static double time_launch(cudaStream_t s, int reps, void (*launch)(cudaStream_t)) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  double best = 1e9, sum = 0;
  for (int i = 0; i < reps + 3; i++) {
    cudaEventRecord(a, s);
    launch(s);
    cudaEventRecord(b, s);
    cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (i >= 3) { sum += ms; if (ms < best) best = ms; }
  }
  printf("best %.2f us mean %.2f us", best * 1e3, sum / reps * 1e3);
  return best;
}
static uint32_t *g_flag;
int main() {
  cudaStream_t s; cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
  cudaMalloc(&g_flag, 4);
  cudaFuncSetAttribute(k_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  printf("== empty kernels, event to event\n");
  printf("<<<1,32>>>                 : "); time_launch(s, 20, [](cudaStream_t st) { k_empty<<<1, 32, 0, st>>>(g_flag); }); printf("\n");
  printf("<<<132,544>>>              : "); time_launch(s, 20, [](cudaStream_t st) { k_empty<<<132, 544, 0, st>>>(g_flag); }); printf("\n");
  printf("<<<132,544>>> 128 B param  : "); time_launch(s, 20, [](cudaStream_t st) { Big b; memset(&b, 1, sizeof(b)); k_empty_big<<<132, 544, 0, st>>>(b, g_flag); }); printf("\n");
  printf("<<<132,544, 64 KB>>>       : "); time_launch(s, 20, [](cudaStream_t st) { k_smem<<<132, 544, 64 * 1024, st>>>(g_flag); }); printf("\n");
  printf("<<<132,544, 199 KB>>>      : "); time_launch(s, 20, [](cudaStream_t st) { k_smem<<<132, 544, 199 * 1024, st>>>(g_flag); }); printf("\n");
  printf("<<<132,544, 199 KB>>> x2 (two back to back between the events): ");
  time_launch(s, 20, [](cudaStream_t st) { k_smem<<<132, 544, 199 * 1024, st>>>(g_flag); k_smem<<<132, 544, 199 * 1024, st>>>(g_flag); }); printf("\n");
  printf("<<<132,544,199 KB>>> after <<<.., 0 KB>>> (carve-out switch): ");
  time_launch(s, 20, [](cudaStream_t st) { k_empty<<<132, 544, 0, st>>>(g_flag); k_smem<<<132, 544, 199 * 1024, st>>>(g_flag); }); printf("\n");
  printf("events only                : "); time_launch(s, 20, [](cudaStream_t) {}); printf("\n");

  const size_t N = 64u << 20, M = 24u << 20;
  uint8_t *d, *hp, *hq; uint8_t *pageable = (uint8_t *)malloc(N);
  cudaMalloc(&d, N + M); cudaMallocHost(&hp, N); cudaMallocHost(&hq, M);
  memset(pageable, 3, N); memset(hp, 1, N); memset(hq, 2, M);
  cudaStream_t s2; cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking);
  auto wall = [](auto f) { auto t0 = std::chrono::steady_clock::now(); f(); return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); };
  printf("== copy engine (64 MiB in, 24 MiB out)\n");
  for (int rep = 0; rep < 2; rep++) {
    double t = wall([&] { cudaMemcpyAsync(d, hp, N, cudaMemcpyHostToDevice, s); cudaStreamSynchronize(s); });
    printf("H2D pinned %.1f GB/s | ", N / t / 1e9);
    t = wall([&] { cudaMemcpyAsync(hq, d + N, M, cudaMemcpyDeviceToHost, s); cudaStreamSynchronize(s); });
    printf("D2H pinned %.1f GB/s | ", M / t / 1e9);
    t = wall([&] { cudaMemcpyAsync(d, hp, N, cudaMemcpyHostToDevice, s); cudaMemcpyAsync(hq, d + N, M, cudaMemcpyDeviceToHost, s2); cudaStreamSynchronize(s); cudaStreamSynchronize(s2); });
    printf("both at once: %.2f ms (H2D alone would be %.2f) | ", t * 1e3, N / 55e9 * 1e3);
    t = wall([&] { cudaMemcpyAsync(d, pageable, N, cudaMemcpyHostToDevice, s); cudaStreamSynchronize(s); });
    printf("H2D pageable %.1f GB/s\n", N / t / 1e9);
  }
  printf("== H2D pinned in chunks (one cudaMemcpyAsync each, queued back to back)\n");
  for (size_t chunk : {size_t(256) << 10, size_t(1) << 20, size_t(2) << 20, size_t(4) << 20, size_t(16) << 20}) {
    double t = wall([&] { for (size_t o = 0; o < N; o += chunk) cudaMemcpyAsync(d + o, hp + o, chunk, cudaMemcpyHostToDevice, s); cudaStreamSynchronize(s); });
    printf("chunk %5zu KiB: %.1f GB/s\n", chunk >> 10, N / t / 1e9);
  }
  printf("== kernel stores to mapped host memory (24 MiB, 16-byte vectors)\n");
  uint4 *hq_dev = nullptr;
  cudaHostGetDevicePointer((void **)&hq_dev, hq, 0);
  for (int grid : {8, 32, 132}) {
    double t = wall([&] { k_store_host<<<grid, 256, 0, s>>>(hq_dev, M / 16); cudaStreamSynchronize(s); });
    t = wall([&] { k_store_host<<<grid, 256, 0, s>>>(hq_dev, M / 16); cudaStreamSynchronize(s); });
    printf("grid %3d: %.1f GB/s | ", grid, M / t / 1e9);
    t = wall([&] { cudaMemcpyAsync(d, hp, N, cudaMemcpyHostToDevice, s2); k_store_host<<<grid, 256, 0, s>>>(hq_dev, M / 16); cudaStreamSynchronize(s); cudaStreamSynchronize(s2); });
    printf("with a 64 MiB H2D alongside: %.2f ms\n", t * 1e3);
  }
  printf("== memcpy pageable -> pinned, T threads (64 MiB)\n");
  for (int T : {1, 2, 4, 6, 8, 12, 16, 32}) {
    double best = 1e9;
    for (int rep = 0; rep < 4; rep++) {
      double t = wall([&] {
        std::vector<std::thread> th;
        for (int i = 0; i < T; i++) th.emplace_back([&, i] { size_t per = N / T; memcpy(hp + i * per, pageable + i * per, per); });
        for (auto &x : th) x.join();
      });
      if (t < best) best = t;
    }
    printf("T=%2d: %.1f GB/s\n", T, N / best / 1e9);
  }
  printf("hardware threads: %u\n", std::thread::hardware_concurrency());
  return 0;
}
