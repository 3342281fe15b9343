// Plain streaming-read rate of the card (the denominator for the pipeline kernels' HBM fraction): every thread reads int4
// vectors of an 8 GB buffer with a grid-stride loop; best of 10 launches by CUDA events, at 4 / 8 / 16 CTAs of 512 per SM.
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o /tmp/stream_read scripts/stream_read.cu && /tmp/stream_read
#include <cstdio>
#include <cuda_runtime.h>

__global__ void sum_kernel(const int4* __restrict__ p, size_t n, unsigned long long* out) {
  unsigned s = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int4 v = __ldcs(p + i);
    s += v.x ^ v.y ^ v.z ^ v.w;
  }
  if (s == 0x12345678u) atomicAdd(out, 1ull);
}

int main() {
  const size_t bytes = 8ull << 30, n = bytes / 16;
  int4* p; unsigned long long* out;
  cudaMalloc(&p, bytes); cudaMalloc(&out, 8);
  cudaMemset(p, 1, bytes);
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int blocks_per_sm : {4, 8, 16}) {
    const int grid = sms * blocks_per_sm;
    for (int w = 0; w < 2; ++w) sum_kernel<<<grid, 512>>>(p, n, out);
    float best = 1e30f;
    for (int r = 0; r < 10; ++r) {
      cudaEventRecord(a); sum_kernel<<<grid, 512>>>(p, n, out); cudaEventRecord(b); cudaEventSynchronize(b);
      float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms;
    }
    printf("{\"blocks_per_sm\": %d, \"ms_best\": %.3f, \"GBps\": %.1f}\n", blocks_per_sm, best, bytes / best / 1e6);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
  cudaFree(p); cudaFree(out);
  return 0;
}
