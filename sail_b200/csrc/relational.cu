// relational.cu -- kernels behind HashJoinExec (multi-match path), SortExec/TopK and row gathers.
//
//   * join_count / join_emit : duplicate-key build sides (HashJoinExec general case): per probe row
//     walk the open-addressing run, count then emit (build row, probe row) pairs.  The unique-key
//     fast path never comes here: it runs inside the tile pipeline (OP_PROBE, pipeline.cu).
//   * sort_encode + radix passes : SortExec.  Rows are encoded into order-preserving fixed-width keys
//     (arrow-row style: null byte, sign-flipped big-endian integers, IEEE total order, strings as their
//     dense rank) and sorted by a stable LSD radix sort on 8-bit digits whose per-warp ranking uses
//     __match_any_sync / ballots ("radix sort via warp shuffles", BASELINE.json north_star).
//   * string_ranks : the dense memcmp-order rank of every string of a column, by MSD refinement of
//     8-byte windows, so that a string key encodes in 4 bytes whatever its length.
//   * gather_rows : `take` of fixed-width / view columns by row index.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "dev_util.cuh"
#include "kernels.hpp"
#include "relational.hpp"

namespace sg {

// ------------------------------------------------------------------------------------------------
// raw-column key hashing: must equal pack_key() in pipeline.cu (the build sink hashes VM slots)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool col_is_null(const RawKeyCol& k, int64_t row) {
  return k.validity_bits && !((k.validity_bits[row >> 3] >> (row & 7)) & 1);
}
__device__ __forceinline__ uint64_t raw_key_hash(const RawKeyCol* keys, int n_keys, int64_t row, bool* has_null) {
  uint64_t h = 0x243F6A8885A308D3ull;
  *has_null = false;
  for (int i = 0; i < n_keys; ++i) {
    const RawKeyCol& k = keys[i];
    if (col_is_null(k, row)) { *has_null = true; return 0; }
    const uint8_t* p = k.data + row * k.stride;
    if (k.width == 16) {
      ulonglong2 v = *reinterpret_cast<const ulonglong2*>(p);
      h = mix64(h ^ (k.is_view ? view_hash(v) : mix64(v.x ^ mix64(v.y))));
    } else {
      uint64_t v = k.width == 8 ? *reinterpret_cast<const uint64_t*>(p) : k.width == 4 ? (uint64_t)*reinterpret_cast<const uint32_t*>(p) : (uint64_t)*p;
      h = mix64(h ^ v);
    }
  }
  return h;
}
__device__ __forceinline__ bool raw_keys_equal(const RawKeyCol* a, int64_t ra, const RawKeyCol* b, int64_t rb, int n_keys) {
  for (int i = 0; i < n_keys; ++i) {
    const uint8_t* pa = a[i].data + ra * a[i].stride;
    const uint8_t* pb = b[i].data + rb * b[i].stride;
    if (a[i].width == 16) {
      ulonglong2 x = *reinterpret_cast<const ulonglong2*>(pa), y = *reinterpret_cast<const ulonglong2*>(pb);
      if (a[i].is_view ? !view_equal(x, y) : (x.x != y.x || x.y != y.y)) return false;
    } else if (a[i].width == 8) { if (*reinterpret_cast<const uint64_t*>(pa) != *reinterpret_cast<const uint64_t*>(pb)) return false; }
    else if (a[i].width == 4) { if (*reinterpret_cast<const uint32_t*>(pa) != *reinterpret_cast<const uint32_t*>(pb)) return false; }
    else if (*pa != *pb) return false;
  }
  return true;
}

// pass 0: counts[i] = number of build rows matching probe row i.  pass 1: write pairs at offs[i].
__global__ void join_multi_kernel(JoinMultiParams P) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P.n_probe; i += (int64_t)gridDim.x * blockDim.x) {
    bool has_null;
    const uint64_t h = raw_key_hash(P.probe_keys, P.n_keys, i, &has_null);
    uint32_t n = 0;
    uint64_t out = P.pass == 1 ? P.offsets[i] : 0;
    if (!has_null) {
      const uint64_t tag = h | 1ull;
      uint64_t idx = (h >> 1) & P.capacity_mask;
      for (;;) {
        const ulonglong2 s = *reinterpret_cast<const ulonglong2*>(P.table + idx * 16);
        if (s.x == 0) break;
        if (s.x == tag && raw_keys_equal(P.build_keys, (int64_t)s.y - 1, P.probe_keys, i, P.n_keys)) {      // slot head = row + 1
          for (int64_t b = (int64_t)s.y - 1; b >= 0; b = P.next[b]) {      // every build row with this key
            if (P.pass == 1) { P.out_build[out] = b; P.out_probe[out] = i; ++out; }
            if (P.pass >= 1 && P.visited) P.visited[b] = 1;            // pass 2 = mark only (semi / anti joins emitting build rows)
            ++n;
          }
          break;                                                        // one slot per distinct key
        }
        idx = (idx + 1) & P.capacity_mask;
      }
    }
    if (P.pass == 0) {
      P.counts[i] = (P.emit_unmatched_probe && n == 0) ? 1u : n;
    } else if (P.pass == 1 && P.emit_unmatched_probe && n == 0) {
      P.out_build[out] = -1; P.out_probe[out] = i;
    }
  }
}

cudaError_t launch_join_multi(const JoinMultiParams& P, cudaStream_t s) {
  if (P.n_probe == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((P.n_probe + 255) / 256, grid_cap(16));
  join_multi_kernel<<<grid, 256, 0, s>>>(P);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// gather (take)
// ------------------------------------------------------------------------------------------------
__global__ void gather_rows_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, const int64_t* __restrict__ idx, int64_t n, int width) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx[i];
    if (width == 16) { ulonglong2 v; v.x = 0; v.y = 0; if (r >= 0) v = *reinterpret_cast<const ulonglong2*>(src + r * 16); *reinterpret_cast<ulonglong2*>(dst + i * 16) = v; }
    else if (width == 8) *reinterpret_cast<uint64_t*>(dst + i * 8) = r >= 0 ? *reinterpret_cast<const uint64_t*>(src + r * 8) : 0;
    else if (width == 4) *reinterpret_cast<uint32_t*>(dst + i * 4) = r >= 0 ? *reinterpret_cast<const uint32_t*>(src + r * 4) : 0;
    else if (width == 2) *reinterpret_cast<uint16_t*>(dst + i * 2) = r >= 0 ? *reinterpret_cast<const uint16_t*>(src + r * 2) : 0;
    else dst[i] = r >= 0 ? src[r] : 0;
  }
}
cudaError_t launch_gather_rows(const uint8_t* src, uint8_t* dst, const int64_t* idx, int64_t n, int width, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(16));
  gather_rows_kernel<<<grid, 256, 0, s>>>(src, dst, idx, n, width);
  return cudaGetLastError();
}
// bit column gathered into bytes: out[i] = bit(src, idx[i]) (0 when idx < 0 or src == null -> `dflt`)
__global__ void gather_bits_kernel(const uint8_t* __restrict__ bits, uint8_t* __restrict__ out, const int64_t* __restrict__ idx, int64_t n, int dflt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx[i];
    out[i] = r < 0 ? 0 : (bits ? (bits[r >> 3] >> (r & 7)) & 1 : dflt);
  }
}
cudaError_t launch_gather_bits(const uint8_t* bits, uint8_t* out, const int64_t* idx, int64_t n, int dflt, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(16));
  gather_bits_kernel<<<grid, 256, 0, s>>>(bits, out, idx, n, dflt);
  return cudaGetLastError();
}
__global__ void iota_kernel(int64_t* out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = i;
}
__global__ void widen_u32_kernel(const uint32_t* in, int64_t* out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = in[i];
}

// ------------------------------------------------------------------------------------------------
// sort: key encoding
// ------------------------------------------------------------------------------------------------
__global__ void max_view_len_kernel(const ulonglong2* views, int64_t n, unsigned int* out) {
  unsigned int m = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = max(m, (unsigned int)views[i].x);
  for (int d = 16; d; d >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, d));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}
cudaError_t launch_max_view_len(const void* views, int64_t n, unsigned int* out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  max_view_len_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const ulonglong2*>(views), n, out);
  return cudaGetLastError();
}

// Encodes every row into `key_bytes` order-preserving bytes (memcmp order == sort order) and, on the way, records
// per byte position which bits were ever set / ever clear (P.bits_or / P.bits_nand): a position where no bit was
// both set and clear is constant over the input and its radix pass is skipped.
__global__ void sort_encode_kernel(SortEncodeParams P) {
  extern __shared__ uint32_t sh_bits[];            // [0, kb): or, [kb, 2kb): nand
  const int kb = P.key_bytes;
  for (int b = threadIdx.x; b < 2 * kb; b += blockDim.x) sh_bits[b] = 0;
  __syncthreads();
#define SG_PUT(pos, val)                                                                 \
  do {                                                                                   \
    const int p_ = (pos); const uint32_t v_ = (uint8_t)(val);                            \
    out[p_] = (uint8_t)v_;                                                               \
    if (v_ & ~sh_bits[p_]) atomicOr(&sh_bits[p_], v_);                                   \
    if ((v_ ^ 0xFFu) & ~sh_bits[kb + p_]) atomicOr(&sh_bits[kb + p_], v_ ^ 0xFFu);       \
  } while (0)
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P.n; i += (int64_t)gridDim.x * blockDim.x) {
    uint8_t* out = P.keys + i * kb;
    for (int k = 0; k < P.n_keys; ++k) {
      const SortKeyCol& c = P.cols[k];
      int o = c.out_off;
      const bool isnull = c.validity_bits && !((c.validity_bits[i >> 3] >> (i & 7)) & 1);
      SG_PUT(o, isnull ? (c.nulls_first ? 0x00 : 0xFF) : (c.nulls_first ? 0x01 : 0x00));
      ++o;
      const uint8_t inv = c.asc ? 0x00 : 0xFF;
      const int w = c.enc_bytes;
      if (isnull) { for (int b = 0; b < w; ++b) SG_PUT(o + b, 0); continue; }
      switch (c.kind) {
        case SORT_INT:        // signed integer of c.width bytes -> big endian, sign bit flipped
        case SORT_UINT: {
          const uint8_t* p = c.data + i * c.width;
          for (int b = 0; b < c.width; ++b) SG_PUT(o + b, p[c.width - 1 - b] ^ inv ^ ((b == 0 && c.kind == SORT_INT) ? 0x80 : 0x00));
          break;
        }
        case SORT_F64: {      // IEEE-754 total order
          uint64_t v = *reinterpret_cast<const uint64_t*>(c.data + i * 8);
          v = (v >> 63) ? ~v : (v | 0x8000000000000000ull);
          for (int b = 0; b < 8; ++b) SG_PUT(o + b, (uint8_t)(v >> (56 - 8 * b)) ^ inv);
          break;
        }
        case SORT_BOOL: {
          const uint8_t v = (c.data[i >> 3] >> (i & 7)) & 1;
          SG_PUT(o, v ^ inv);
          break;
        }
        default: {            // SORT_VIEW: the string's dense rank (launch_string_ranks), 4 bytes big-endian
          const uint32_t r = c.rank[i];
          for (int b = 0; b < 4; ++b) SG_PUT(o + b, (uint8_t)(r >> (24 - 8 * b)) ^ inv);
        }
      }
    }
  }
#undef SG_PUT
  __syncthreads();
  for (int b = threadIdx.x; b < 2 * kb; b += blockDim.x)
    if (sh_bits[b]) atomicOr(P.bits + b, sh_bits[b]);
}
cudaError_t launch_sort_encode(const SortEncodeParams& P, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((P.n + 255) / 256, grid_cap(8));
  sort_encode_kernel<<<grid, 256, (size_t)P.key_bytes * 8, s>>>(P);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// sort: stable LSD radix sort of (key word, row index) pairs, 8-bit digits.
// The encoded key is consumed 8 bytes at a time from its least significant end: the 8 bytes of every row are
// gathered once (in the current order) into a u64 that then travels with the row index through the passes of
// that word, so a pass reads and writes only sequential / bucket-contiguous 12 B records.  Digits that are
// constant over the input (see sort_encode_kernel) cost nothing.  Each warp owns RADIX_CHUNK consecutive records.
// ------------------------------------------------------------------------------------------------
constexpr int RADIX_CHUNK = 2048;

__global__ void radix_gather_word_kernel(const uint8_t* __restrict__ keys, int key_bytes, int lo, int nb, const uint32_t* __restrict__ idx, int64_t n,
                                         uint64_t* __restrict__ kw) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t* p = keys + (int64_t)(idx ? idx[i] : (uint32_t)i) * key_bytes + lo;
    uint64_t v = 0;
    for (int b = 0; b < nb; ++b) v = (v << 8) | p[b];
    kw[i] = v;
  }
}

__global__ void radix_hist_kernel(const uint64_t* __restrict__ kw, int shift, int64_t n, uint32_t* __restrict__ hist /* [256][n_chunks] */, int64_t n_chunks) {
  const int lane = threadIdx.x & 31;
  const int64_t chunk = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (chunk >= n_chunks) return;
  __shared__ uint32_t sh[8][256];
  uint32_t* h = sh[(threadIdx.x >> 5)];
  for (int b = lane; b < 256; b += 32) h[b] = 0;
  __syncwarp();
  const int64_t b0 = chunk * RADIX_CHUNK, b1 = min(n, b0 + RADIX_CHUNK);
  for (int64_t i = b0 + lane; i < b1; i += 32) atomicAdd(&h[(kw[i] >> shift) & 255u], 1u);
  __syncwarp();
  for (int b = lane; b < 256; b += 32) hist[(int64_t)b * n_chunks + chunk] = h[b];
}

__global__ void radix_scatter_kernel(const uint64_t* __restrict__ kw_in, const uint32_t* __restrict__ idx_in, uint64_t* __restrict__ kw_out,
                                     uint32_t* __restrict__ idx_out, int shift, int64_t n, const uint64_t* __restrict__ offs /* scanned hist */,
                                     int64_t n_chunks) {
  const int lane = threadIdx.x & 31;
  const int64_t chunk = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (chunk >= n_chunks) return;
  __shared__ uint64_t sh[8][256];
  uint64_t* base = sh[(threadIdx.x >> 5)];
  for (int b = lane; b < 256; b += 32) base[b] = offs[(int64_t)b * n_chunks + chunk];
  __syncwarp();
  const int64_t b0 = chunk * RADIX_CHUNK, b1 = min(n, b0 + RADIX_CHUNK);
  for (int64_t g = b0; g < b1; g += 32) {
    const int64_t i = g + lane;
    const bool in = i < b1;
    const uint64_t w = in ? kw_in[i] : 0;
    const uint32_t row = in ? (idx_in ? idx_in[i] : (uint32_t)i) : 0;
    const uint32_t d = in ? (uint32_t)((w >> shift) & 255u) : 0x100u + lane;   // idle lanes match nobody
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, d);
    const int rank = __popc(peers & ((1u << lane) - 1));
    uint64_t pos = 0;
    if (in) pos = base[d] + rank;
    __syncwarp();
    if (in && rank == __popc(peers) - 1) base[d] += __popc(peers);   // last peer advances the cursor
    __syncwarp();
    if (in) { kw_out[pos] = w; idx_out[pos] = row; }
  }
}

__global__ void iota_u32_kernel(uint32_t* out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (uint32_t)i;
}

// n <= 1024: one CTA ranks every row against every other (stable: ties broken by input position)
__global__ void small_sort_kernel(const uint8_t* __restrict__ keys, int key_bytes, int n, uint32_t* __restrict__ idx_out) {
  const int i = threadIdx.x;
  if (i >= n) return;
  const uint8_t* ki = keys + (int64_t)i * key_bytes;
  int rank = 0;
  for (int j = 0; j < n; ++j) {
    const uint8_t* kj = keys + (int64_t)j * key_bytes;
    int c = 0;
    for (int b = 0; b < key_bytes && c == 0; ++b) c = (int)kj[b] - (int)ki[b];
    rank += (c < 0 || (c == 0 && j < i)) ? 1 : 0;
  }
  idx_out[rank] = (uint32_t)i;
}

// n <= 1024 without an encoding pass: one CTA ranks every row against every other by comparing the key columns in place,
// in exactly the order sort_encode_kernel's bytes give (stable: ties broken by input position).  Strings are compared as
// they are, so no bound on their length has to be known beforehand.
__device__ int cmp_sort_key(const SortKeyCol& c, int64_t a, int64_t b) {
  const bool na = c.validity_bits && !((c.validity_bits[a >> 3] >> (a & 7)) & 1);
  const bool nb = c.validity_bits && !((c.validity_bits[b >> 3] >> (b & 7)) & 1);
  if (na || nb) return na == nb ? 0 : ((na == (c.nulls_first != 0)) ? -1 : 1);
  int r = 0;
  switch (c.kind) {
    case SORT_INT:
    case SORT_UINT: {        // most significant byte first, sign bit flipped for signed integers
      const uint8_t* pa = c.data + a * c.width;
      const uint8_t* pb = c.data + b * c.width;
      for (int i = 0; i < c.width && r == 0; ++i) {
        const uint8_t f = (i == 0 && c.kind == SORT_INT) ? 0x80 : 0x00;
        r = (int)(pa[c.width - 1 - i] ^ f) - (int)(pb[c.width - 1 - i] ^ f);
      }
      break;
    }
    case SORT_F64: {
      uint64_t x = *reinterpret_cast<const uint64_t*>(c.data + a * 8), y = *reinterpret_cast<const uint64_t*>(c.data + b * 8);
      x = (x >> 63) ? ~x : (x | 0x8000000000000000ull);
      y = (y >> 63) ? ~y : (y | 0x8000000000000000ull);
      r = x < y ? -1 : (x > y ? 1 : 0);
      break;
    }
    case SORT_BOOL:
      r = (int)((c.data[a >> 3] >> (a & 7)) & 1) - (int)((c.data[b >> 3] >> (b & 7)) & 1);
      break;
    default: {               // SORT_VIEW: bytes, the shorter string padded with zeros, then the length
      const uint8_t* va = c.data + a * 16;
      const uint8_t* vb = c.data + b * 16;
      const ulonglong2 x = *reinterpret_cast<const ulonglong2*>(va), y = *reinterpret_cast<const ulonglong2*>(vb);
      const uint32_t la = (uint32_t)x.x, lb = (uint32_t)y.x;
      const uint8_t* sa = view_ptr(x, va);
      const uint8_t* sb = view_ptr(y, vb);
      const uint32_t m = la > lb ? la : lb;
      for (uint32_t i = 0; i < m && r == 0; ++i) r = (int)(i < la ? sa[i] : 0) - (int)(i < lb ? sb[i] : 0);
      if (r == 0) r = la < lb ? -1 : (la > lb ? 1 : 0);
    }
  }
  return c.asc ? r : -r;
}
__global__ void small_sort_cols_kernel(const SortEncodeParams P, uint32_t* __restrict__ idx_out) {
  const int i = threadIdx.x;
  if (i >= P.n) return;
  int rank = 0;
  for (int j = 0; j < (int)P.n; ++j) {
    int c = 0;
    for (int k = 0; k < P.n_keys && c == 0; ++k) c = cmp_sort_key(P.cols[k], j, i);
    rank += (c < 0 || (c == 0 && j < i)) ? 1 : 0;
  }
  idx_out[rank] = (uint32_t)i;
}
cudaError_t launch_small_sort_cols(const SortEncodeParams& P, uint32_t* idx_out, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  if (P.n > SMALL_SORT_ROWS) return cudaErrorInvalidValue;
  small_sort_cols_kernel<<<1, SMALL_SORT_ROWS, 0, s>>>(P, idx_out);
  return cudaGetLastError();
}

// Sorts row indices by the encoded keys; `S.idx_a` receives the final order.  `bits` = the [2 * key_bytes] words
// sort_encode_kernel filled.  Synchronises the stream once (to read `bits`).  *launches counts the kernels issued.
cudaError_t radix_sort_indices(const uint8_t* keys, int key_bytes, int64_t n, const RadixScratch& S, const uint32_t* bits, cudaStream_t s, int* launches) {
  if (launches) *launches = 0;
  if (n == 0) return cudaSuccess;
  std::vector<uint32_t> hb((size_t)key_bytes * 2);
  if (n > 1024) {
    cudaError_t e = cudaMemcpyAsync(hb.data(), bits, hb.size() * 4, cudaMemcpyDeviceToHost, s);
    if (e != cudaSuccess) return e;
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return e;
  }
  return radix_sort_indices_host_bits(keys, key_bytes, n, S, hb.data(), s, launches);
}
// the same with `hb` = those words already on the host: no synchronisation
cudaError_t radix_sort_indices_host_bits(const uint8_t* keys, int key_bytes, int64_t n, const RadixScratch& S, const uint32_t* hb, cudaStream_t s, int* launches) {
  int nl = 0;
  if (launches) *launches = 0;
  if (n == 0) return cudaSuccess;
  if (n <= 1024) { small_sort_kernel<<<1, 1024, 0, s>>>(keys, key_bytes, (int)n, S.idx_a); if (launches) *launches = 1; return cudaGetLastError(); }
  cudaError_t e = cudaSuccess;
  auto trivial = [&](int d) { return (hb[(size_t)d] & hb[(size_t)key_bytes + d] & 0xFFu) == 0; };
  const int64_t n_chunks = (n + RADIX_CHUNK - 1) / RADIX_CHUNK;
  const int blocks = (int)((n_chunks + 7) / 8);
  const int flat = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  const uint32_t* in_idx = nullptr;            // nullptr = identity order
  uint32_t* out_idx = S.idx_a;
  uint64_t* kw_in = S.kw_a; uint64_t* kw_out = S.kw_b;
  for (int hi = key_bytes; hi > 0;) {
    const int lo = std::max(0, hi - 8);
    bool any = false;
    for (int d = lo; d < hi; ++d) any |= !trivial(d);
    if (any) {
      radix_gather_word_kernel<<<flat, 256, 0, s>>>(keys, key_bytes, lo, hi - lo, in_idx, n, kw_in); ++nl;
      for (int d = hi - 1; d >= lo; --d) {
        if (trivial(d)) continue;
        const int shift = 8 * (hi - 1 - d);
        radix_hist_kernel<<<blocks, 256, 0, s>>>(kw_in, shift, n, S.hist, n_chunks);
        e = launch_exclusive_scan_u32(S.hist, 256 * n_chunks, S.offs, S.scan_scratch, s);
        if (e != cudaSuccess) return e;
        radix_scatter_kernel<<<blocks, 256, 0, s>>>(kw_in, in_idx, kw_out, out_idx, shift, n, S.offs, n_chunks);
        nl += 5;
        std::swap(kw_in, kw_out);
        in_idx = out_idx;
        out_idx = (out_idx == S.idx_a) ? S.idx_b : S.idx_a;
      }
    }
    hi = lo;
  }
  if (in_idx == nullptr) { iota_u32_kernel<<<flat, 256, 0, s>>>(S.idx_a, n); ++nl; }
  else if (in_idx != S.idx_a) { e = cudaMemcpyAsync(S.idx_a, in_idx, (size_t)n * 4, cudaMemcpyDeviceToDevice, s); if (e != cudaSuccess) return e; }
  if (launches) *launches = nl;
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// string ranks: the dense rank of every string of a Utf8View column in memcmp order (a proper prefix before its extensions).
// MSD refinement: round r orders the rows of every open group by (group, the 8 bytes of the string at 8r big-endian and
// zero-padded, marker = min(bytes left, 9)) with the radix sort above and writes them back into their group's positions.
// A group is open while it has two or more rows and its strings go on past the window (marker 9).  A row leaves as soon as
// its group is settled: it pays for the windows it shares with another row, not for the longest string of the column.
// Null rows rank as the empty string (the encoding's null byte decides their place).
// ------------------------------------------------------------------------------------------------
constexpr int RANK_KEY = 13;          // 4 B group, 8 B window, 1 B marker
constexpr uint32_t RANK_WIN = 8;

__device__ __forceinline__ void rank_bits_put(uint32_t* bits, int pos, uint32_t o, uint32_t a) {
  if (o) atomicOr(bits + pos, o);
  if (a != 0xFFu) atomicOr(bits + RANK_KEY + pos, a ^ 0xFFu);
}
// the round's key of every open row (count ? *count : n of them); records which key bits vary, as sort_encode_kernel does
__global__ void rank_encode_kernel(const uint8_t* __restrict__ views, const uint8_t* __restrict__ validity, int64_t n, const uint32_t* __restrict__ count,
                                   uint32_t offset, const uint32_t* __restrict__ opos, const uint32_t* __restrict__ grp, const uint32_t* __restrict__ perm,
                                   uint32_t* __restrict__ rowof, uint8_t* __restrict__ keys, uint32_t* __restrict__ bits) {
  const int64_t m = count ? (int64_t)*count : n;
  uint32_t og = 0, ag = 0xFFFFFFFFu, om = 0, am = 0xFFu;
  uint64_t ow = 0, aw = ~0ull;
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < m; j += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t row = opos ? perm[opos[j]] : (uint32_t)j;
    if (opos) rowof[j] = row;
    const uint32_t g = grp ? grp[j] : 0u;
    const uint8_t* vp = views + (int64_t)row * 16;
    const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(vp);
    const bool valid = !validity || ((validity[row >> 3] >> (row & 7)) & 1);
    const uint32_t rest = (valid ? (uint32_t)v.x : 0u) - offset;       // the rows of an open group go on past `offset`
    const uint8_t* sp = view_ptr(v, vp) + offset;
    const uint32_t nb = rest < RANK_WIN ? rest : RANK_WIN;
    uint64_t w = 0;
    for (uint32_t b = 0; b < nb; ++b) w |= (uint64_t)sp[b] << (56 - 8 * b);
    const uint32_t mk = rest < RANK_WIN + 1 ? rest : RANK_WIN + 1;
    uint8_t* k = keys + j * RANK_KEY;
    for (int b = 0; b < 4; ++b) k[b] = (uint8_t)(g >> (24 - 8 * b));
    for (int b = 0; b < 8; ++b) k[4 + b] = (uint8_t)(w >> (56 - 8 * b));
    k[12] = (uint8_t)mk;
    og |= g; ag &= g; ow |= w; aw &= w; om |= mk; am &= mk;
  }
  for (int d = 16; d; d >>= 1) {
    og |= __shfl_xor_sync(0xFFFFFFFFu, og, d); ag &= __shfl_xor_sync(0xFFFFFFFFu, ag, d);
    ow |= __shfl_xor_sync(0xFFFFFFFFu, ow, d); aw &= __shfl_xor_sync(0xFFFFFFFFu, aw, d);
    om |= __shfl_xor_sync(0xFFFFFFFFu, om, d); am &= __shfl_xor_sync(0xFFFFFFFFu, am, d);
  }
  if ((threadIdx.x & 31) == 0) {
    for (int b = 0; b < 4; ++b) rank_bits_put(bits, b, (og >> (24 - 8 * b)) & 0xFFu, (ag >> (24 - 8 * b)) & 0xFFu);
    for (int b = 0; b < 8; ++b) rank_bits_put(bits, 4 + b, (uint32_t)(ow >> (56 - 8 * b)) & 0xFFu, (uint32_t)(aw >> (56 - 8 * b)) & 0xFFu);
    rank_bits_put(bits, 12, om, am);
  }
}
__device__ __forceinline__ bool rank_key_eq(const uint8_t* a, const uint8_t* b) {
  for (int i = 0; i < RANK_KEY; ++i) if (a[i] != b[i]) return false;
  return true;
}
// the sorted open rows back into their groups' positions; new group heads; flags[i] = open row | (first row of an open group) << 32
__global__ void rank_refine_kernel(const uint8_t* __restrict__ keys, const uint32_t* __restrict__ idx, int64_t m, const uint32_t* __restrict__ opos,
                                   const uint32_t* __restrict__ rowof, uint32_t* __restrict__ perm, uint32_t* __restrict__ head, uint64_t* __restrict__ flags) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t j = idx[i];
    const uint8_t* kj = keys + (int64_t)j * RANK_KEY;
    const uint32_t p = opos ? opos[i] : (uint32_t)i;
    perm[p] = rowof ? rowof[j] : j;
    const bool eq_prev = i > 0 && rank_key_eq(kj, keys + (int64_t)idx[i - 1] * RANK_KEY);
    const bool eq_next = i + 1 < m && rank_key_eq(kj, keys + (int64_t)idx[i + 1] * RANK_KEY);
    if (!eq_prev) head[p] = 1u;
    const bool open = kj[12] == RANK_WIN + 1 && (eq_prev || eq_next);
    flags[i] = (uint64_t)open | ((uint64_t)(open && !eq_prev) << 32);
  }
}
// the open rows of the next round: their positions and dense open-group numbers (in position order); *count = how many
__global__ void rank_compact_kernel(const uint64_t* __restrict__ flags, const uint64_t* __restrict__ before, int64_t m, const uint32_t* __restrict__ opos,
                                    uint32_t* __restrict__ opos_out, uint32_t* __restrict__ grp_out, uint32_t* __restrict__ count) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t f = flags[i], b = before[i];      // low half: open rows before i; high half: open groups begun before i
    if (f & 1u) {
      opos_out[(uint32_t)b] = opos ? opos[i] : (uint32_t)i;
      grp_out[(uint32_t)b] = (uint32_t)(b >> 32) + (uint32_t)(f >> 32) - 1u;
    }
    if (i == m - 1) *count = (uint32_t)b + (uint32_t)f;
  }
}
__global__ void rank_assign_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ head, const uint64_t* __restrict__ before, int64_t n,
                                   uint32_t* __restrict__ rank) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
    rank[perm[p]] = (uint32_t)(before[p] + head[p] - 1u);
}

cudaError_t string_ranks(const void* views, const uint8_t* validity, int64_t n, uint32_t* rank, const StringRankScratch& S, cudaStream_t s, int* launches,
                         int* syncs) {
  int nl = 0, ns = 0;
  *launches = 0; *syncs = 0;
  if (n == 0) return cudaSuccess;
  auto grid = [](int64_t m) { return (int)std::min<int64_t>((m + 255) / 256, grid_cap(8)); };
  const uint8_t* vw = static_cast<const uint8_t*>(views);
  uint32_t* count = S.ctrl + 2 * RANK_KEY;
  uint32_t hc[2 * RANK_KEY + 1];
  cudaError_t e = cudaMemsetAsync(S.head, 0, (size_t)n * 4, s);
  if (e != cudaSuccess) return e;
  const uint32_t *opos = nullptr, *grp = nullptr;
  int64_t m = n;                       // open rows of the round (an upper bound until the read-back)
  for (uint32_t offset = 0, buf = 0;; offset += RANK_WIN, buf ^= 1) {
    if ((e = cudaMemsetAsync(S.ctrl, 0, 2 * RANK_KEY * 4, s)) != cudaSuccess) return e;
    rank_encode_kernel<<<grid(m), 256, 0, s>>>(vw, validity, n, offset ? count : nullptr, offset, opos, grp, S.perm, S.rowof, S.keys, S.ctrl);
    ++nl;
    // the one read-back of the round: how many rows are open, and which key bytes vary among them
    if ((e = cudaMemcpyAsync(hc, S.ctrl, sizeof(hc), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
    ++ns;
    if (offset) m = hc[2 * RANK_KEY];
    if (m == 0) break;
    int sl = 0;
    if ((e = radix_sort_indices_host_bits(S.keys, RANK_KEY, m, S.radix, hc, s, &sl)) != cudaSuccess) return e;
    rank_refine_kernel<<<grid(m), 256, 0, s>>>(S.keys, S.radix.idx_a, m, opos, opos ? S.rowof : nullptr, S.perm, S.head, S.flags);
    if ((e = launch_exclusive_scan_u64(S.flags, m, S.before, S.scan_scratch, s)) != cudaSuccess) return e;
    rank_compact_kernel<<<grid(m), 256, 0, s>>>(S.flags, S.before, m, opos, S.opos[buf], S.grp[buf], count);
    nl += sl + 5;
    opos = S.opos[buf]; grp = S.grp[buf];
  }
  if ((e = launch_exclusive_scan_u32(S.head, n, S.before, S.scan_scratch, s)) != cudaSuccess) return e;
  rank_assign_kernel<<<grid(n), 256, 0, s>>>(S.perm, S.head, S.before, n, rank);
  nl += 4;
  *launches = nl; *syncs = ns;
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// TopK selection (SortExec with fetch = k, test_tpch.plan.yaml:27,79; ClickBench ORDER BY .. LIMIT 10): radix SELECT on
// a 64-bit word per row instead of sorting all n rows.  One level = one streaming pass over 8 B/row: histogram of the next
// 11 bits among the rows whose consumed prefix equals the threshold path.
// ------------------------------------------------------------------------------------------------
// The word is the leading 8 bytes of the order-preserving encoding, built from the key columns, except that a string key
// contributes its own leading bytes (zero-padded, inverted when descending) and nothing comes after it.  It is monotone in the
// requested order (a < b implies word(a) <= word(b)), which is all the selection needs; the candidates are then sorted exactly.
__global__ void topk_word_kernel(const SortEncodeParams P, uint64_t* __restrict__ words) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P.n; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t w = 0;
    int pos = 0;
    auto put = [&](uint32_t b) { if (pos < 8) w |= (uint64_t)(b & 0xFFu) << (56 - 8 * pos); ++pos; };
    for (int k = 0; k < P.n_keys && pos < 8; ++k) {
      const SortKeyCol& c = P.cols[k];
      const bool isnull = c.validity_bits && !((c.validity_bits[i >> 3] >> (i & 7)) & 1);
      put(isnull ? (c.nulls_first ? 0x00 : 0xFF) : (c.nulls_first ? 0x01 : 0x00));
      const uint32_t inv = c.asc ? 0x00 : 0xFF;
      if (c.kind == SORT_VIEW) {
        if (!isnull) {
          const uint8_t* vp = c.data + i * 16;
          const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(vp);
          const uint32_t len = (uint32_t)v.x;
          const uint8_t* s = view_ptr(v, vp);
          for (uint32_t b = 0; pos < 8; ++b) put((b < len ? s[b] : 0u) ^ inv);
        }
        break;
      }
      if (isnull) { pos += c.enc_bytes; continue; }
      switch (c.kind) {
        case SORT_INT:
        case SORT_UINT: {
          const uint8_t* p = c.data + i * c.width;
          for (int b = 0; b < c.width && pos < 8; ++b) put(p[c.width - 1 - b] ^ inv ^ ((b == 0 && c.kind == SORT_INT) ? 0x80u : 0x00u));
          break;
        }
        case SORT_F64: {
          uint64_t v = *reinterpret_cast<const uint64_t*>(c.data + i * 8);
          v = (v >> 63) ? ~v : (v | 0x8000000000000000ull);
          for (int b = 0; b < 8 && pos < 8; ++b) put((uint32_t)(v >> (56 - 8 * b)) ^ inv);
          break;
        }
        default:              // SORT_BOOL
          put(((c.data[i >> 3] >> (i & 7)) & 1u) ^ inv);
      }
    }
    words[i] = w;
  }
}
cudaError_t launch_topk_words(const SortEncodeParams& P, uint64_t* words, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  topk_word_kernel<<<(int)std::min<int64_t>((P.n + 255) / 256, grid_cap(8)), 256, 0, s>>>(P, words);
  return cudaGetLastError();
}
__global__ void topk_hist_kernel(const uint64_t* __restrict__ words, int64_t n, int used, uint64_t prefix, int digit_bits, uint32_t* __restrict__ hist) {
  __shared__ uint32_t sh[2048];
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t w = words[i];
    if (used == 0 || (w >> (64 - used)) == prefix) atomicAdd(&sh[(uint32_t)((w << used) >> (64 - digit_bits))], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) if (sh[i]) atomicAdd(&hist[i], sh[i]);
}
// rows whose leading `used` word bits are <= threshold (every row when used == 0): their indices, in any order
__global__ void topk_compact_kernel(const uint64_t* __restrict__ words, int64_t n, int used, uint64_t threshold, int64_t* __restrict__ out, unsigned long long* counter) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t w = words[i];
    const bool take = used == 0 || (w >> (64 - used)) <= threshold;
    const unsigned m = __ballot_sync(__activemask(), take);
    if (take) {
      const unsigned lane = threadIdx.x & 31;
      const int lead = __ffs(m) - 1;
      unsigned long long base = 0;
      if ((int)lane == lead) base = atomicAdd(counter, (unsigned long long)__popc(m));
      base = __shfl_sync(m, base, lead);
      out[base + __popc(m & ((1u << lane) - 1))] = i;
    }
  }
}
cudaError_t launch_topk_hist(const uint64_t* words, int64_t n, int used, uint64_t prefix, int digit_bits, uint32_t* hist, cudaStream_t s) {
  topk_hist_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(words, n, used, prefix, digit_bits, hist);
  return cudaGetLastError();
}
cudaError_t launch_topk_compact(const uint64_t* words, int64_t n, int used, uint64_t threshold, int64_t* out, unsigned long long* counter, cudaStream_t s) {
  topk_compact_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(words, n, used, threshold, out, counter);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// k-way merge of sorted runs (SortPreservingMergeExec, test_tpch.plan.yaml:9-10): every row computes its output position
// directly -- its index in its own run plus, for every other run, the number of rows that sort before it (binary search
// on the encoded keys; ties go to the earlier run, which makes the merge stable).  No sequential merge loop, no heap.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int key_cmp(const uint8_t* a, const uint8_t* b, int key_bytes) {
  for (int i = 0; i < key_bytes; ++i) { const int d = (int)a[i] - (int)b[i]; if (d) return d; }
  return 0;
}
__global__ void merge_rank_kernel(const uint8_t* __restrict__ keys, int key_bytes, const int64_t* __restrict__ run_off, int n_runs, int64_t n, int64_t* __restrict__ perm) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int r = 0;
    while (r + 1 < n_runs && run_off[r + 1] <= i) ++r;      // (runs are few)
    const uint8_t* me = keys + i * key_bytes;
    int64_t pos = i - run_off[r];
    for (int s = 0; s < n_runs; ++s) {
      if (s == r) continue;
      int64_t lo = run_off[s], hi = run_off[s + 1];
      while (lo < hi) {          // s < r: rows <= me sort first (upper bound); s > r: rows < me (lower bound)
        const int64_t mid = (lo + hi) >> 1;
        const int c = key_cmp(keys + mid * key_bytes, me, key_bytes);
        if (c < 0 || (c == 0 && s < r)) lo = mid + 1; else hi = mid;
      }
      pos += lo - run_off[s];
    }
    perm[pos] = i;
  }
}
cudaError_t launch_merge_rank(const uint8_t* keys, int key_bytes, const int64_t* run_off, int n_runs, int64_t n, int64_t* perm, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  merge_rank_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(keys, key_bytes, run_off, n_runs, n, perm);
  return cudaGetLastError();
}

// sort-based grouping (aggregates whose group key does not fit the hash table's packed key).  Rows are ordered by a 64-bit hash of
// their key columns (8 radix digits whatever the key width; strings hashed whole, NULL a value of its own); `heads` marks the
// first row of every run of equal keys (cmp_sort_key == 0 on every column).  Two different keys with one hash would make equal
// keys non-adjacent: *collisions counts adjacent rows with equal hash and different keys, and the caller then orders by the key.
__global__ void group_hash_kernel(const SortEncodeParams P, uint8_t* __restrict__ out8) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P.n; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t h = 0x243F6A8885A308D3ull;
    for (int k = 0; k < P.n_keys; ++k) {
      const SortKeyCol& c = P.cols[k];
      if (c.validity_bits && !((c.validity_bits[i >> 3] >> (i & 7)) & 1)) { h = mix64(h ^ 0x9E3779B97F4A7C15ull); continue; }
      if (c.kind == SORT_VIEW) { h = mix64(h ^ view_hash(*reinterpret_cast<const ulonglong2*>(c.data + i * 16))); continue; }
      if (c.kind == SORT_BOOL) { h = mix64(h ^ ((c.data[i >> 3] >> (i & 7)) & 1u)); continue; }
      const uint8_t* p = c.data + i * c.width;
      for (int j = 0; j < c.width; j += 8) {
        uint64_t w = 0;
        for (int b = 0; b < 8 && j + b < c.width; ++b) w |= (uint64_t)p[j + b] << (8 * b);
        h = mix64(h ^ w);
      }
    }
    for (int b = 0; b < 8; ++b) out8[i * 8 + b] = (uint8_t)(h >> (56 - 8 * b));      // big-endian: memcmp order == numeric order
  }
}
cudaError_t launch_group_hash(const SortEncodeParams& P, uint8_t* out8, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  group_hash_kernel<<<(int)std::min<int64_t>((P.n + 255) / 256, grid_cap(8)), 256, 0, s>>>(P, out8);
  return cudaGetLastError();
}
__global__ void group_heads_kernel(const SortEncodeParams P, const uint32_t* __restrict__ idx, uint32_t* __restrict__ heads,
                                   const uint64_t* __restrict__ hashes, unsigned long long* __restrict__ collisions) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P.n; i += (int64_t)gridDim.x * blockDim.x) {
    bool head = i == 0;
    if (i > 0) {
      for (int k = 0; k < P.n_keys && !head; ++k) head = cmp_sort_key(P.cols[k], idx[i], idx[i - 1]) != 0;
      if (head && hashes && hashes[idx[i]] == hashes[idx[i - 1]]) atomicAdd(collisions, 1ull);
    }
    heads[i] = head ? 1u : 0u;
  }
}
cudaError_t launch_group_heads(const SortEncodeParams& P, const uint32_t* idx, uint32_t* heads, const uint8_t* hashes, unsigned long long* collisions, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  group_heads_kernel<<<(int)std::min<int64_t>((P.n + 255) / 256, grid_cap(8)), 256, 0, s>>>(P, idx, heads, reinterpret_cast<const uint64_t*>(hashes), collisions);
  return cudaGetLastError();
}
// group number of every input row (dense, in key order) and one representative input row per group
__global__ void assign_groups_kernel(const uint32_t* __restrict__ idx, const uint32_t* __restrict__ heads, const uint64_t* __restrict__ before, int64_t n,
                                     int64_t* __restrict__ gid_of_row, int64_t* __restrict__ rep) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = (int64_t)before[i] + (int64_t)heads[i] - 1;      // heads before i, plus this one
    gid_of_row[idx[i]] = g;
    if (heads[i]) rep[g] = (int64_t)idx[i];
  }
}
cudaError_t launch_assign_groups(const uint32_t* idx, const uint32_t* heads, const uint64_t* before, int64_t n, int64_t* gid_of_row, int64_t* rep, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  assign_groups_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(idx, heads, before, n, gid_of_row, rep);
  return cudaGetLastError();
}

cudaError_t launch_iota(int64_t* out, int64_t n, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  iota_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(out, n);
  return cudaGetLastError();
}
__global__ void iota_stride_kernel(int64_t* out, int64_t first, int64_t stride, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = first + i * stride;
}
cudaError_t launch_iota_stride(int64_t* out, int64_t first, int64_t stride, int64_t n, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  iota_stride_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(out, first, stride, n);
  return cudaGetLastError();
}
cudaError_t launch_widen_u32(const uint32_t* in, int64_t* out, int64_t n, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  widen_u32_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(in, out, n);
  return cudaGetLastError();
}

// rebases resolved views by a constant delta (exchange: received heap segment vs sender heap)
__global__ void rebase_views_kernel(ulonglong2* views, int64_t n, uint64_t heap_base) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    ulonglong2 v = views[i];
    if ((uint32_t)v.x > 12) { v.y = heap_base + (v.y >> 32); views[i] = v; }   // Arrow view: offset in the high half
  }
}
cudaError_t launch_rebase_views(void* views, int64_t n, uint64_t heap_base, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  rebase_views_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(reinterpret_cast<ulonglong2*>(views), n, heap_base);
  return cudaGetLastError();
}

}  // namespace sg
