// kernels.hpp -- host-callable launchers implemented in the .cu files.
#pragma once
#include <cuda_runtime.h>

#include "vm.h"

namespace sg {

// Grid of a grid-stride launch: at most `per_sm` CTAs on every SM of the current device.
inline int grid_cap(int per_sm) {
  static const int sms = [] {
    int d = 0, n = 0;
    if (cudaGetDevice(&d) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d) != cudaSuccess || n <= 0) n = 132;
    return n;
  }();
  return sms * per_sm;
}

struct AggOutCol {
  int32_t kind;        // 0 group key i, 1 accumulator state/final j, 2 avg(sum acc j, count acc k), 3-5 variance (compiler.hpp AggOutSpec)
  int32_t a, b, c;
  int32_t var;         // kind 5: VAR_POP | VAR_SQRT
  int32_t width;
  int32_t src_words;
  int32_t key_word;
  int32_t is_float;
  int32_t nullable;
  uint64_t scale_mul_lo, scale_mul_hi;
  uint8_t* data;
  uint8_t* valid_bytes;
};
struct AggExtractParams {
  int32_t n_cols;
  AggOutCol cols[MAX_KEYS + 2 * MAX_ACCS];
};

// Carrying a group table over to a wider entry layout (a later batch brought validity buffers an earlier one lacked):
// where every word of a new entry comes from in the old one.
struct AggMigrateMap {
  int32_t old_entry_words, old_key_words;
  int32_t key_shift;                 // 1: the new layout gained the leading null-mask word
  int32_t pad;
  int16_t acc_src_word[MAX_ACCS];    // first word (inside the old accumulator area) of the accumulator a new one continues
  int8_t seen_src[MAX_ACCS];         // old accumulator index whose seen bit carries over; -1: every old contribution was valid (bit set); -2: not tracked
};
cudaError_t launch_agg_migrate(const AggParams& A_new, const AggMigrateMap& M, const uint8_t* old_table, const uint32_t* old_occ, uint64_t old_groups, uint32_t* err, cudaStream_t s);
cudaError_t launch_pipeline(const KernelArgs& K, int rpt, int n_stages, size_t smem_bytes, int grid, int minb, cudaStream_t stream);
int pipeline_max_ctas_per_sm(int rpt, int minb, size_t smem_bytes, int sink, bool cold);
cudaError_t launch_tile_popcount(const uint32_t* bits, int64_t n_rows, int tile_rows, int64_t n_tiles, uint32_t* counts, cudaStream_t s);
cudaError_t launch_agg_rehash(const AggParams& A, const uint8_t* old_table, const uint32_t* old_occ, uint64_t old_groups, uint32_t* err, cudaStream_t s);
cudaError_t launch_agg_extract(const AggParams& A, const AggExtractParams& X, uint64_t n_groups, uint32_t* err, cudaStream_t s);
cudaError_t launch_pack_bytes(const uint8_t* bytes, uint32_t* bits, int64_t n, unsigned long long* null_count, cudaStream_t s);
cudaError_t launch_u32_to_bytes(const uint32_t* in, uint8_t* out, int64_t n, cudaStream_t s);
cudaError_t launch_unpack_bits(const uint8_t* bits, uint8_t* bytes, int64_t n, int64_t bit_offset, cudaStream_t s);
cudaError_t launch_resolve_views(void* views, int64_t n, const uint64_t* bases, cudaStream_t s);
cudaError_t launch_utf8_to_views(const int32_t* offsets, const uint8_t* bytes, void* views, int64_t n, cudaStream_t s);
cudaError_t launch_exclusive_scan_u32(const uint32_t* in, int64_t n, uint64_t* out, uint64_t* block_scratch, cudaStream_t s);
cudaError_t launch_exclusive_scan_u64(const uint64_t* in, int64_t n, uint64_t* out, uint64_t* block_scratch, cudaStream_t s);
cudaError_t launch_view_lengths(const void* views, int64_t n, uint32_t* lens, int all, cudaStream_t s);
cudaError_t launch_views_to_arrow(void* views, int64_t n, const uint64_t* offs, uint8_t* heap, cudaStream_t s);
cudaError_t launch_views_to_utf8(const void* views, int64_t n, const uint64_t* offs, int32_t* out_offsets, uint8_t* heap, cudaStream_t s);

// sort.cu
cudaError_t launch_gather_rows(const uint8_t* src, uint8_t* dst, const int64_t* idx, int64_t n, int width, cudaStream_t s);

}  // namespace sg
