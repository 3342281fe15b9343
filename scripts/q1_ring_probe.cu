// Load-path probe for the specialised aggregate kernel (jit_rt.cuh jit_main): Q1's input traffic -- seven column streams of
// 16, 16, 16, 16, 16, 16 and 4 B/row, 100 B/row over 64 Mi rows (6.7 GB) -- fed through variants of the TMA stage ring, each
// consuming its tile with a clock64 spin that stands in for Q1's arithmetic.  One JSON line per variant; the plain
// streaming read of scripts/stream_read.cu runs in the same process as the denominator.
//
//   producer "thread0": thread 0 of warp 0 waits until every warp released tile it-1, refills that stage, then consumes (jit_main)
//   producer "warp":    a ninth warp only produces; the eight consumer warps never wait for it
//   producer "poll":    thread 0 refills every released stage while it waits for its own next tile (try_wait, never blocks)
//   rows_per_stage 512: two 256-row tiles per stage, consumed one after the other (one row live per thread)
//   "plain":            no staging, every thread loads its row with 16-byte (and one 4-byte) ld.global.nc
//
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o /tmp/q1_ring_probe scripts/q1_ring_probe.cu && /tmp/q1_ring_probe
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#include "../sail_b200/csrc/dev_util.cuh"

using namespace sg;

constexpr int NT = 256, NWARPS = NT / 32, NCOL = 7;
__host__ __device__ constexpr int width(int c) { return c < NCOL - 1 ? 16 : 4; }
constexpr int ROW_BYTES = 100;
constexpr int HDR = 256;
constexpr int SCRATCH = 4608;                 // Q1's dictionary scratch, so that CTAs per SM match the real kernel
constexpr int64_t N_ROWS = 64ll << 20;

struct Cols { const uint8_t* p[NCOL]; };

__device__ __forceinline__ uint32_t consume_row(const uint8_t* st, int rows, int r) {
  uint32_t acc = 0, off = 0;
#pragma unroll
  for (int c = 0; c < NCOL; ++c) {
    if (width(c) == 16) { const uint4 v = *reinterpret_cast<const uint4*>(st + off + r * 16); acc ^= v.x ^ v.y ^ v.z ^ v.w; }
    else acc ^= *reinterpret_cast<const uint32_t*>(st + off + r * 4);
    off += width(c) * rows;
  }
  return acc;
}
__device__ __forceinline__ void spin_until(long long t0, long long cycles) { while (clock64() - t0 < cycles) {} }

enum { P_THREAD0 = 0, P_WARP = 1, P_POLL = 2 };

template <int S, int MODE, int H>
__global__ void __launch_bounds__(NT + 32) ring_kernel(Cols c, long long spin, unsigned long long* out) {
  constexpr int ROWS = 256 * H;
  constexpr uint32_t STAGE = ROW_BYTES * ROWS;
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + S;
  long long* tile_no = reinterpret_cast<long long*>(empty + S);
  uint8_t* ring = smem + HDR + SCRATCH;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t n_tiles = N_ROWS / ROWS;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NWARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  auto produce = [&](int64_t j) {
    const int s = (int)(j % S);
    const int64_t tn = blockIdx.x + j * gridDim.x;
    uint8_t* st = ring + (size_t)s * STAGE;
    if (tn < n_tiles) {
      tile_no[s] = tn;
      fence_proxy_async();
      mbar_expect_tx(&full[s], STAGE);
      uint32_t off = 0;
      for (int k = 0; k < NCOL; ++k) { tma_load_1d(st + off, c.p[k] + tn * ROWS * width(k), width(k) * ROWS, &full[s]); off += width(k) * ROWS; }
    } else {
      tile_no[s] = -1;
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&full[s])) : "memory");
    }
    return tn < n_tiles;
  };
  if (MODE == P_WARP) {
    if (warp == NWARPS) {
      if (lane == 0)
        for (int64_t j = 0;; ++j) {
          if (j >= S) mbar_wait(&empty[j % S], (uint32_t)(((j - S) / S) & 1));
          if (!produce(j)) break;
        }
      return;
    }
  } else if (tid == 0) {
    for (int j = 0; j < S - 1; ++j) produce(j);
  }
  int64_t prod = S - 1;           // P_POLL: next ring position thread 0 fills
  bool done = false;
  uint32_t acc = 0;
  for (int64_t it = 0;; ++it) {
    const int s = (int)(it % S);
    const uint32_t ph = (uint32_t)((it / S) & 1);
    if (MODE == P_THREAD0 && tid == 0) {
      if (it >= 1) mbar_wait(&empty[(it - 1) % S], (uint32_t)(((it - 1) / S) & 1));
      produce(it + S - 1);
    }
    if (MODE == P_POLL && tid == 0) {
      for (uint32_t spins = 0;; ++spins) {
        while (!done && prod <= it + S - 1 && (prod < S || mbar_try_wait(&empty[prod % S], (uint32_t)(((prod - S) / S) & 1)))) done = !produce(prod++);
        if (mbar_try_wait(&full[s], ph)) break;
        if (spins > (1u << 26)) __trap();
      }
    }
    __syncwarp();
    mbar_wait(&full[s], ph);
    __syncwarp();
    if (tile_no[s] < 0) break;
    const uint8_t* st = ring + (size_t)s * STAGE;
#pragma unroll
    for (int h = 0; h < H; ++h) {
      const long long t0 = clock64();
      acc ^= consume_row(st, ROWS, tid + h * NT);
      spin_until(t0, spin);
    }
    __syncwarp();
    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[s])) : "memory");
  }
  if (acc == 0x12345678u) atomicAdd(out, 1ull);
}

__global__ void __launch_bounds__(NT) plain_kernel(Cols c, long long spin, unsigned long long* out) {
  uint32_t acc = 0;
  const int64_t n_tiles = N_ROWS / NT;
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int64_t r = t * NT + threadIdx.x;
    const long long t0 = clock64();
    uint4 v[NCOL - 1];
#pragma unroll
    for (int k = 0; k < NCOL - 1; ++k) v[k] = __ldg(reinterpret_cast<const uint4*>(c.p[k]) + r);
    uint32_t d = __ldg(reinterpret_cast<const uint32_t*>(c.p[NCOL - 1]) + r);
#pragma unroll
    for (int k = 0; k < NCOL - 1; ++k) d ^= v[k].x ^ v[k].y ^ v[k].z ^ v[k].w;
    acc ^= d;
    spin_until(t0, spin);
  }
  if (acc == 0x12345678u) atomicAdd(out, 1ull);
}

__global__ void stream_kernel(const int4* __restrict__ p, size_t n, unsigned long long* out) {      // scripts/stream_read.cu
  unsigned s = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int4 v = __ldcs(p + i);
    s += v.x ^ v.y ^ v.z ^ v.w;
  }
  if (s == 0x12345678u) atomicAdd(out, 1ull);
}

static cudaEvent_t ev_a, ev_b;
template <class F> static float best_ms(F launch) {
  for (int w = 0; w < 2; ++w) launch();
  float best = 1e30f;
  for (int r = 0; r < 5; ++r) {
    cudaEventRecord(ev_a); launch(); cudaEventRecord(ev_b); cudaEventSynchronize(ev_b);
    float ms; cudaEventElapsedTime(&ms, ev_a, ev_b); if (ms < best) best = ms;
  }
  return best;
}

static Cols g_cols;
static unsigned long long* g_out;
static int g_sms;
static double g_stream_tbps;
static const long long kSpins[] = {0, 500, 1000, 1500, 2000, 3000};

static void report(const char* variant, const char* producer, int stages, int rows, int ctas, long long spin, float ms) {
  const double tbps = (double)N_ROWS * ROW_BYTES / ms / 1e9;
  printf("{\"variant\": \"%s\", \"producer\": \"%s\", \"stages\": %d, \"rows_per_stage\": %d, \"ctas_per_sm\": %d, \"spin_cycles\": %lld, "
         "\"ms_best\": %.3f, \"TBps\": %.3f, \"of_stream\": %.3f}\n", variant, producer, stages, rows, ctas, spin, ms, tbps, tbps / g_stream_tbps);
  fflush(stdout);
}

template <int S, int MODE, int H> static void run_ring(const char* variant, int ctas) {
  auto k = ring_kernel<S, MODE, H>;
  const int smem = HDR + SCRATCH + S * ROW_BYTES * 256 * H;
  const int nt = NT + (MODE == P_WARP ? 32 : 0);
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  int occ = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, nt, smem);
  if (occ < ctas) return;                 // does not fit at this many CTAs per SM
  static const char* names[] = {"thread0", "warp", "poll"};
  for (long long spin : kSpins) {
    const float ms = best_ms([&] { k<<<g_sms * ctas, nt, smem>>>(g_cols, spin, g_out); });
    report(variant, names[MODE], S, 256 * H, ctas, spin, ms);
  }
}

int main() {
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  g_sms = prop.multiProcessorCount;
  cudaEventCreate(&ev_a); cudaEventCreate(&ev_b);
  cudaMalloc(&g_out, 8);
  uint8_t* buf[NCOL];
  for (int k = 0; k < NCOL; ++k) { cudaMalloc(&buf[k], (size_t)N_ROWS * width(k)); cudaMemset(buf[k], k + 1, (size_t)N_ROWS * width(k)); g_cols.p[k] = buf[k]; }
  {
    const size_t bytes = 8ull << 30, n = bytes / 16;
    int4* p; cudaMalloc(&p, bytes); cudaMemset(p, 1, bytes);
    float best = 1e30f;
    for (int bps : {4, 8, 16}) { const float ms = best_ms([&] { stream_kernel<<<g_sms * bps, 512>>>(p, n, g_out); }); if (ms < best) best = ms; }
    g_stream_tbps = bytes / best / 1e9;
    cudaFree(p);
    printf("{\"device\": \"%s\", \"sms\": %d, \"stream_read_TBps\": %.3f, \"rows\": %lld, \"bytes\": %lld}\n", prop.name, g_sms, g_stream_tbps,
           (long long)N_ROWS, (long long)N_ROWS * ROW_BYTES);
  }
  run_ring<2, P_THREAD0, 1>("a", 2); run_ring<3, P_THREAD0, 1>("a", 2); run_ring<4, P_THREAD0, 1>("a", 2);
  run_ring<2, P_WARP, 1>("b", 2); run_ring<3, P_WARP, 1>("b", 2); run_ring<4, P_WARP, 1>("b", 2);
  run_ring<5, P_WARP, 1>("b", 1); run_ring<6, P_WARP, 1>("b", 1);
  run_ring<2, P_POLL, 1>("b", 2); run_ring<3, P_POLL, 1>("b", 2); run_ring<4, P_POLL, 1>("b", 2);
  run_ring<5, P_POLL, 1>("b", 1); run_ring<6, P_POLL, 1>("b", 1);
  run_ring<2, P_THREAD0, 2>("c", 2); run_ring<2, P_POLL, 2>("c", 2); run_ring<2, P_WARP, 2>("c", 2);
  run_ring<3, P_POLL, 2>("c", 1);
  run_ring<2, P_THREAD0, 1>("d", 1); run_ring<2, P_THREAD0, 1>("d", 3); run_ring<2, P_THREAD0, 1>("d", 4);
  run_ring<2, P_POLL, 1>("d", 3); run_ring<2, P_POLL, 1>("d", 4);
  for (int ctas : {2, 3, 4, 8})
    for (long long spin : kSpins) report("e", "plain", 0, 256, ctas, spin, best_ms([&] { plain_kernel<<<g_sms * ctas, NT>>>(g_cols, spin, g_out); }));
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("{\"error\": \"%s\"}\n", cudaGetErrorString(e)); return 1; }
  for (int k = 0; k < NCOL; ++k) cudaFree(buf[k]);
  cudaFree(g_out);
  return 0;
}
