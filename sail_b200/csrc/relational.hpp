// relational.hpp -- parameter blocks and launchers of relational.cu
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vm.h"

namespace sg {

struct RawKeyCol {
  const uint8_t* data;
  const uint8_t* validity_bits;   // Arrow bitmap or null
  int32_t width;                  // bytes compared / hashed: 1, 4, 8, 16
  int32_t is_view;
  int32_t stride;                 // bytes between rows (16 for a <=18-digit decimal keyed on its low word)
  int32_t pad;
};

struct JoinMultiParams {
  int64_t n_probe;
  int32_t n_keys;
  int32_t pass;                   // 0 count, 1 emit
  int32_t emit_unmatched_probe;   // right-outer: a probe row without match yields (-1, row)
  int32_t pad;
  RawKeyCol probe_keys[MAX_KEYS];
  RawKeyCol build_keys[MAX_KEYS];
  const uint8_t* table;
  uint64_t capacity_mask;
  uint32_t* counts;
  const uint64_t* offsets;
  int64_t* out_build;
  int64_t* out_probe;
  uint8_t* visited;
  const int64_t* next;            // duplicate-key chains built by the build sink
};

enum SortKind : int32_t { SORT_INT = 0, SORT_UINT = 1, SORT_F64 = 2, SORT_BOOL = 3, SORT_VIEW = 4 };
struct SortKeyCol {
  const uint8_t* data;
  const uint8_t* validity_bits;
  int32_t kind, width;
  int32_t asc, nulls_first;
  int32_t out_off;                // offset of this key inside the encoded row
  int32_t enc_bytes;              // value bytes after the null byte
  const uint32_t* rank;           // SORT_VIEW, encoded sort: the dense rank of every row's string (string_ranks)
};
struct SortEncodeParams {
  int64_t n;
  int32_t n_keys, key_bytes;
  uint8_t* keys;
  uint32_t* bits;                 // [2 * key_bytes], zeroed: per byte position the OR of the bytes, then the OR of their complements
  SortKeyCol cols[8];
};
struct RadixScratch {
  uint32_t *idx_a, *idx_b;        // [n]
  uint64_t *kw_a, *kw_b;          // [n]
  uint32_t* hist;                 // [256 * ceil(n / 2048)]
  uint64_t* offs;                 // [256 * ceil(n / 2048)]
  uint64_t* scan_scratch;         // [1026]
};
struct StringRankScratch {
  RadixScratch radix;             // for n rows
  uint8_t* keys;                  // [13 * n]
  uint32_t *perm, *head, *rowof;  // [n]
  uint32_t *opos[2], *grp[2];     // [n]
  uint64_t *flags, *before;       // [n]
  uint64_t* scan_scratch;         // [1026]
  uint32_t* ctrl;                 // [27]
};

cudaError_t launch_join_multi(const JoinMultiParams& P, cudaStream_t s);
cudaError_t launch_gather_bits(const uint8_t* bits, uint8_t* out, const int64_t* idx, int64_t n, int dflt, cudaStream_t s);
cudaError_t launch_max_view_len(const void* views, int64_t n, unsigned int* out, cudaStream_t s);
cudaError_t launch_sort_encode(const SortEncodeParams& P, cudaStream_t s);
// P.n <= SMALL_SORT_ROWS rows ordered by the key columns of P (no `keys` / `bits` needed): idx_out[rank] = row
constexpr int SMALL_SORT_ROWS = 1024;
cudaError_t launch_small_sort_cols(const SortEncodeParams& P, uint32_t* idx_out, cudaStream_t s);
cudaError_t radix_sort_indices(const uint8_t* keys, int key_bytes, int64_t n, const RadixScratch& S, const uint32_t* bits, cudaStream_t s, int* launches);
cudaError_t radix_sort_indices_host_bits(const uint8_t* keys, int key_bytes, int64_t n, const RadixScratch& S, const uint32_t* host_bits, cudaStream_t s, int* launches);
// rank[row] = dense rank of the row's string among the n views (memcmp order, a prefix before its extensions; null rows rank as
// ""), for n < 2^32.  Synchronises the stream once per 8-byte window that some group of equal prefixes still spans (*syncs).
cudaError_t string_ranks(const void* views, const uint8_t* validity, int64_t n, uint32_t* rank, const StringRankScratch& S, cudaStream_t s, int* launches,
                         int* syncs);
cudaError_t launch_topk_words(const SortEncodeParams& P, uint64_t* words, cudaStream_t s);
cudaError_t launch_topk_hist(const uint64_t* words, int64_t n, int used, uint64_t prefix, int digit_bits, uint32_t* hist /* [2048], zeroed */, cudaStream_t s);
cudaError_t launch_topk_compact(const uint64_t* words, int64_t n, int used, uint64_t threshold, int64_t* out, unsigned long long* counter, cudaStream_t s);
cudaError_t launch_merge_rank(const uint8_t* keys, int key_bytes, const int64_t* run_off, int n_runs, int64_t n, int64_t* perm, cudaStream_t s);
cudaError_t launch_group_hash(const SortEncodeParams& P, uint8_t* out8, cudaStream_t s);
// heads[i] = 1 where row idx[i] differs from row idx[i - 1] in some key column of P (P.n rows); with `hashes`, *collisions counts
// heads whose 8-byte hash equals the previous row's
cudaError_t launch_group_heads(const SortEncodeParams& P, const uint32_t* idx, uint32_t* heads, const uint8_t* hashes, unsigned long long* collisions, cudaStream_t s);
cudaError_t launch_assign_groups(const uint32_t* idx, const uint32_t* heads, const uint64_t* before, int64_t n, int64_t* gid_of_row, int64_t* rep, cudaStream_t s);
cudaError_t launch_iota(int64_t* out, int64_t n, cudaStream_t s);
cudaError_t launch_iota_stride(int64_t* out, int64_t first, int64_t stride, int64_t n, cudaStream_t s);
cudaError_t launch_widen_u32(const uint32_t* in, int64_t* out, int64_t n, cudaStream_t s);
cudaError_t launch_rebase_views(void* views, int64_t n, uint64_t heap_base, cudaStream_t s);

}  // namespace sg
