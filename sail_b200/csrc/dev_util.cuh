// dev_util.cuh -- sm_90a device helpers: mbarrier + TMA bulk copy, 128-bit integers, hashing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sg {

typedef __int128 i128;
typedef unsigned __int128 u128;

// ---- mbarrier / TMA 1-D bulk copy (cp.async.bulk -> SASS UBLKCP) -------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// bounded wait: a TMA copy that never lands traps the kernel instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t spins = 0; !mbar_try_wait(bar, parity); ++spins)
    if (spins > (1u << 26)) __trap();
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---- typed shared-memory access ----------------------------------------------------------------
template <typename T> __device__ __forceinline__ T lds(const uint8_t* p) { return *reinterpret_cast<const T*>(p); }
template <> __device__ __forceinline__ i128 lds<i128>(const uint8_t* p) {
  ulonglong2 v = *reinterpret_cast<const ulonglong2*>(p);
  return (i128)(((u128)v.y << 64) | v.x);
}
template <typename T> __device__ __forceinline__ void sts(uint8_t* p, T v) { *reinterpret_cast<T*>(p) = v; }
template <> __device__ __forceinline__ void sts<i128>(uint8_t* p, i128 v) {
  ulonglong2 w; w.x = (unsigned long long)(u128)v; w.y = (unsigned long long)((u128)v >> 64);
  *reinterpret_cast<ulonglong2*>(p) = w;
}

// streaming global stores / loads
__device__ __forceinline__ void stg_i128(uint8_t* p, i128 v) {
  ulonglong2 w; w.x = (unsigned long long)(u128)v; w.y = (unsigned long long)((u128)v >> 64);
  *reinterpret_cast<ulonglong2*>(p) = w;
}

// ---- hashing (splitmix64 finalizer; the same function oracle/ops.py mirrors for partition ids) ----
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// A resolved string view: len<=12 -> bytes inline; else {len, prefix, absolute device pointer}
struct View { uint32_t len; uint32_t prefix; uint64_t rest; };
__device__ __forceinline__ View as_view(ulonglong2 v) {
  View w; w.len = (uint32_t)v.x; w.prefix = (uint32_t)(v.x >> 32); w.rest = v.y; return w;
}
__device__ __forceinline__ const uint8_t* view_ptr(const ulonglong2& v, const uint8_t* self_bytes) {
  // self_bytes: address of the 16-byte view itself (inline data starts at +4)
  return ((uint32_t)v.x <= 12) ? self_bytes + 4 : reinterpret_cast<const uint8_t*>(v.y);
}
__device__ __forceinline__ bool view_equal(ulonglong2 a, ulonglong2 b) {
  if (a.x != b.x) return false;                 // len + 4-byte prefix
  uint32_t len = (uint32_t)a.x;
  if (len <= 12) return a.y == b.y;
  const uint8_t* pa = reinterpret_cast<const uint8_t*>(a.y);
  const uint8_t* pb = reinterpret_cast<const uint8_t*>(b.y);
  if (pa == pb) return true;
  for (uint32_t i = 4; i < len; ++i)
    if (pa[i] != pb[i]) return false;
  return true;
}
__device__ __forceinline__ uint64_t view_hash(ulonglong2 a) {
  uint32_t len = (uint32_t)a.x;
  if (len <= 12) return mix64(a.x ^ mix64(a.y));
  const uint8_t* p = reinterpret_cast<const uint8_t*>(a.y);
  uint64_t h = mix64(a.x);
  uint32_t i = 4;
  for (; i + 8 <= len; i += 8) {
    uint64_t w = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) w |= (uint64_t)p[i + k] << (8 * k);
    h = mix64(h ^ w);
  }
  uint64_t w = 0;
  for (int k = 0; i < len; ++i, ++k) w |= (uint64_t)p[i] << (8 * k);
  return mix64(h ^ w);
}

__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// 128-bit compare-and-swap in global memory (PTX atom.cas.b128, sm_90+)
__device__ __forceinline__ u128 atomic_cas_128(void* addr, u128 expected, u128 desired) {
  unsigned long long e0 = (unsigned long long)expected, e1 = (unsigned long long)(expected >> 64);
  unsigned long long d0 = (unsigned long long)desired, d1 = (unsigned long long)(desired >> 64);
  unsigned long long r0, r1;
  asm volatile(
      "{\n"
      ".reg .b128 e, d, r;\n"
      "mov.b128 e, {%2, %3};\n"
      "mov.b128 d, {%4, %5};\n"
      "atom.global.cas.b128 r, [%6], e, d;\n"
      "mov.b128 {%0, %1}, r;\n"
      "}\n"
      : "=l"(r0), "=l"(r1)
      : "l"(e0), "l"(e1), "l"(d0), "l"(d1), "l"(addr)
      : "memory");
  return ((u128)r1 << 64) | r0;
}

}  // namespace sg
