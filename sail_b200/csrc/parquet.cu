// parquet.cu -- Parquet column chunks -> Arrow columns in HBM (SURVEY.md section 8 row f2).
//
// The step before the operator path: Sail's scans are DataFusion `DataSourceExec(ParquetSource)` nodes
// (crates/sail-data-source/src/listing/planner.rs:47, adapted at crates/sail-execution/src/task_runner/core.rs:115-133)
// that decode pages to Arrow on CPU cores; an operator path at TB/s is then fed at the pace of that decode and of PCIe
// moving 16-byte decimals.  Here the column chunk crosses PCIe AS STORED (dictionary indices, 7-byte decimals, ...) and is
// decoded on the device.  The host only walks what is inherently sequential and tiny: Thrift page headers and the run
// headers of the RLE / bit-packed hybrid streams (a few bytes per run); every value is produced by a GPU thread.
//
// Covered: data pages V1 / V2, dictionary pages, PLAIN and RLE_DICTIONARY / PLAIN_DICTIONARY values, DELTA_BINARY_PACKED
// (INT32 / INT64), DELTA_LENGTH_BYTE_ARRAY (BYTE_ARRAY), DELTA_BYTE_ARRAY (BYTE_ARRAY / FIXED_LEN_BYTE_ARRAY) and
// BYTE_STREAM_SPLIT (DOUBLE / INT32 / INT64 / FIXED_LEN_BYTE_ARRAY) values, any mix of them in one chunk, RLE definition levels of
// flat optional columns (max level 1), physical types INT32 / INT64 / DOUBLE / FIXED_LEN_BYTE_ARRAY / BYTE_ARRAY, uncompressed
// and ZSTD-compressed pages.  BOOLEAN, FLOAT and INT96 columns, other codecs and nested columns are refused
// (SAILGPU_ERR_UNSUPPORTED): the caller keeps the CPU reader for those files.  Of the DELTA streams the host walks only the
// block headers (one descriptor per block); one thread per value unpacks its delta and a wrapping 64-bit scan adds them up.
//
// INT32 decodes to Int32 / Date32, to Decimal128, and to the narrow integers Int8 / Int16 / UInt8 / UInt16 (how Parquet stores
// the INT(8|16, signed|unsigned) logical types, e.g. ClickBench's Int16 columns and its UInt16 EventDate): the value kept is the
// low 1 or 2 bytes of the INT32, which is how parquet-cpp and arrow-rs truncate.  BYTE_ARRAY decodes to Utf8View whatever the
// column's annotation: the annotation never reaches this code, so a UTF8 string column and a plain binary one (ClickBench's URL,
// Title, ... read with `binary_as_string`) take the same path.  The bytes are passed through unchanged and are not validated as
// UTF-8; whether Sail's CPU reader rejects invalid UTF-8 in a binary column read as string is not checked here.  INT64 columns
// annotated TIMESTAMP(MILLIS|MICROS|NANOS, isAdjustedToUTC) decode to the Timestamp type the caller names, in the same way: the
// annotation does not reach this code, and the 8-byte values pass through unchanged.  INT96 timestamps stay refused.
//
// ZSTD chunks (Sail's writer default) are decompressed on the device first.  Page headers are stored uncompressed, so the host
// walks them into a page table (where each page's frames start, how long they are, where the decompressed body goes) and
// checks each page's first frame header.  One launch of parquet_zstd_decompress_kernel covers the compressed pages of every
// column of the call, one warp per page (zstd.cuh), and builds a decompressed image of each chunk: every page's header bytes
// followed by its decompressed body (the levels of a data page V2 are stored uncompressed and are copied as they are).  The
// images are read back once, with a status per page, because the run-header walk below runs on the host; from there on a
// ZSTD chunk is its image, already in HBM, and takes the uncompressed path.
#include <cstring>

#include "device.hpp"
#include "h2d.hpp"
#include "kernels.hpp"
#include "zstd.cuh"

namespace sg {

namespace {

// ---- Thrift compact protocol (reader for the page header structs) ---------------------------------
struct TReader {
  const uint8_t* p; const uint8_t* end;
  int16_t last = 0;
  uint64_t varint() {
    uint64_t v = 0; int sh = 0;
    for (;;) {
      SG_CHECK(p < end && sh < 64, SAILGPU_ERR_INVALID, "parquet: truncated page header");
      const uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7F) << sh;
      if (!(b & 0x80)) return v;
      sh += 7;
    }
  }
  int64_t zigzag() { const uint64_t v = varint(); return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }
  // next field of the current struct: false at STOP
  bool field(int* id, int* type) {
    SG_CHECK(p < end, SAILGPU_ERR_INVALID, "parquet: truncated page header");
    const uint8_t b = *p++;
    if (b == 0) return false;
    *type = b & 0x0F;
    const int delta = b >> 4;
    last = delta ? (int16_t)(last + delta) : (int16_t)zigzag();
    *id = last;
    return true;
  }
  void skip(int type) {
    switch (type) {
      case 1: case 2: break;                       // booleans live in the field header
      case 3: ++p; break;
      case 4: case 5: case 6: (void)zigzag(); break;
      case 7: p += 8; break;
      case 8: { const uint64_t n = varint(); p += n; break; }
      case 9: case 10: {
        const uint8_t h = *p++;
        uint64_t n = h >> 4; const int et = h & 0x0F;
        if (n == 15) n = varint();
        for (uint64_t i = 0; i < n; ++i) skip(et);
        break;
      }
      case 12: { const int16_t save = last; last = 0; int id, t; while (field(&id, &t)) skip(t); last = save; break; }
      default: fail(SAILGPU_ERR_UNSUPPORTED, "parquet: page header field type " + std::to_string(type));
    }
    SG_CHECK(p <= end, SAILGPU_ERR_INVALID, "parquet: truncated page header");
  }
};

struct PageHeader {
  int type = -1, uncompressed = 0, compressed = 0;
  int num_values = 0, encoding = -1, def_encoding = 3;
  int num_nulls = -1, def_bytes = 0, rep_bytes = 0; bool v2_compressed = true;
};
enum { PAGE_DATA = 0, PAGE_DICT = 2, PAGE_DATA_V2 = 3 };
enum { ENC_PLAIN = 0, ENC_PLAIN_DICT = 2, ENC_RLE = 3, ENC_DBP = 5, ENC_DLBA = 6, ENC_DBA = 7, ENC_RLE_DICT = 8, ENC_BSS = 9 };
enum { PT_BOOLEAN = 0, PT_INT32 = 1, PT_INT64 = 2, PT_INT96 = 3, PT_FLOAT = 4, PT_DOUBLE = 5, PT_BYTE_ARRAY = 6, PT_FLBA = 7 };

PageHeader read_page_header(TReader& r) {
  PageHeader h;
  r.last = 0;
  int id, t;
  while (r.field(&id, &t)) {
    if (id == 1 && t == 5) h.type = (int)r.zigzag();
    else if (id == 2 && t == 5) h.uncompressed = (int)r.zigzag();
    else if (id == 3 && t == 5) h.compressed = (int)r.zigzag();
    else if ((id == 5 || id == 7 || id == 8) && t == 12) {
      const int16_t save = r.last; r.last = 0;
      int fid, ft;
      while (r.field(&fid, &ft)) {
        if (id == 5) {
          if (fid == 1 && ft == 5) h.num_values = (int)r.zigzag();
          else if (fid == 2 && ft == 5) h.encoding = (int)r.zigzag();
          else if (fid == 3 && ft == 5) h.def_encoding = (int)r.zigzag();
          else r.skip(ft);
        } else if (id == 7) {
          if (fid == 1 && ft == 5) h.num_values = (int)r.zigzag();
          else if (fid == 2 && ft == 5) h.encoding = (int)r.zigzag();
          else r.skip(ft);
        } else {
          if (fid == 1 && ft == 5) h.num_values = (int)r.zigzag();
          else if (fid == 2 && ft == 5) h.num_nulls = (int)r.zigzag();
          else if (fid == 4 && ft == 5) h.encoding = (int)r.zigzag();
          else if (fid == 5 && ft == 5) h.def_bytes = (int)r.zigzag();
          else if (fid == 6 && ft == 5) h.rep_bytes = (int)r.zigzag();
          else if (fid == 7 && (ft == 1 || ft == 2)) h.v2_compressed = ft == 1;
          else r.skip(ft);
        }
      }
      r.last = save;
    } else r.skip(t);
  }
  return h;
}

// ---- RLE / bit-packed hybrid: the host reads the run headers, the device expands the runs ---------
struct Run {
  int64_t out_start;      // first output element
  int64_t src_bit;        // bit-packed: bit offset of the run's first value inside the chunk
  uint32_t count;
  uint32_t value;         // RLE: the repeated value
  uint32_t packed;        // 1: bit-packed
  uint32_t bit_width;
};

// walks a hybrid stream of `n_values` values; appends runs (clipped to n_values); returns the number of values equal to `count_value`
int64_t scan_hybrid(const uint8_t* chunk, const uint8_t* p, const uint8_t* end, int bit_width, int64_t n_values, int64_t out_start, std::vector<Run>* runs,
                    uint32_t count_value) {
  int64_t produced = 0, matches = 0;
  TReader r{p, end};
  const int vbytes = (bit_width + 7) / 8;
  while (produced < n_values) {
    SG_CHECK(r.p < end, SAILGPU_ERR_INVALID, "parquet: RLE stream ends before its page does");
    const uint64_t h = r.varint();
    if (h & 1) {
      const uint64_t groups = h >> 1;
      const int64_t cnt = std::min<int64_t>((int64_t)groups * 8, n_values - produced);
      Run run{out_start + produced, (int64_t)(r.p - chunk) * 8, (uint32_t)cnt, 0, 1, (uint32_t)bit_width};
      runs->push_back(run);
      if (bit_width == 1) {                      // definition levels: count the set bits (how many values the page carries)
        for (int64_t i = 0; i < cnt; ++i) matches += ((r.p[i >> 3] >> (i & 7)) & 1u) == count_value;
      }
      r.p += groups * (uint64_t)bit_width;
      SG_CHECK(r.p <= end, SAILGPU_ERR_INVALID, "parquet: bit-packed run overruns its page");
      produced += cnt;
    } else {
      const int64_t cnt = std::min<int64_t>((int64_t)(h >> 1), n_values - produced);
      uint32_t v = 0;
      SG_CHECK(r.p + vbytes <= end, SAILGPU_ERR_INVALID, "parquet: RLE run overruns its page");
      for (int b = 0; b < vbytes; ++b) v |= (uint32_t)r.p[b] << (8 * b);
      r.p += vbytes;
      if (cnt > 0) runs->push_back(Run{out_start + produced, 0, (uint32_t)cnt, v, 0, (uint32_t)bit_width});
      if (v == count_value) matches += cnt;
      produced += cnt;
    }
  }
  return matches;
}

__global__ void expand_runs_kernel(const uint8_t* __restrict__ chunk, const Run* __restrict__ runs, const int64_t* __restrict__ run_start, int n_runs, int64_t n,
                                   uint32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = n_runs - 1;                 // last run whose start <= i
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (run_start[mid] <= i) lo = mid; else hi = mid - 1; }
    const Run r = runs[lo];
    uint32_t v = r.value;
    if (r.packed) {
      const int64_t bit = r.src_bit + (i - r.out_start) * (int64_t)r.bit_width;
      uint64_t w = 0;
      const uint8_t* p = chunk + (bit >> 3);
#pragma unroll
      for (int b = 0; b < 5; ++b) w |= (uint64_t)p[b] << (8 * b);            // 32 value bits + 7 bits of offset fit in 5 bytes (buffers are padded)
      v = (uint32_t)((w >> (bit & 7)) & ((r.bit_width >= 32) ? 0xFFFFFFFFull : ((1ull << r.bit_width) - 1)));
    }
    out[i] = v;
  }
}

// ---- DELTA_* and BYTE_STREAM_SPLIT pages -> PLAIN layout in a per-column buffer ------------------------------------------
// Values of these pages are numbered in the column's "decoded" space: the non-null values of its DELTA / BYTE_STREAM_SPLIT
// pages, in page order.  They are decoded into one buffer, in PLAIN layout (4 / 8 / type_length bytes, or ready 16-byte
// views for strings), which decode_values_kernel then reads like a PLAIN page.
constexpr uint32_t ERR_CORRUPT_STREAM = 1u << 8;     // error flag: a DELTA stream the host could not check is corrupt

// One block of a DELTA_BINARY_PACKED stream, walked on the host.  The thread of decoded value i unpacks the delta that leads
// to the stream's next value, so the stream's values are first_value + an exclusive scan of the deltas.
struct DeltaBlock {
  int64_t start;                  // decoded index whose thread unpacks the block's first delta
  int64_t first, last;            // decoded indices of the stream's first and last value
  uint64_t first_value, min_delta;
  uint64_t widths_off, mb_off;    // chunk offsets of the block's miniblock bit widths and of its first miniblock
  uint64_t per_mb;                // values per miniblock
};
// one DELTA / BYTE_STREAM_SPLIT data page in decoded space; data_off / data_len: the BYTE_STREAM_SPLIT values, or the bytes
// after the length streams of a DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY page
struct DecPage { int64_t first, count; uint64_t data_off, data_len; int64_t encoding; };

template <typename T, int64_t T::*Start>
__device__ __forceinline__ int last_at_or_before(const T* v, int n, int64_t i) {   // last entry that starts at or before i (or 0)
  int lo = 0, hi = n - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (v[mid].*Start <= i) lo = mid; else hi = mid - 1; }
  return lo;
}

__global__ void delta_unpack_kernel(const uint8_t* __restrict__ chunk, const DeltaBlock* __restrict__ blocks, int n_blocks, int64_t n, uint64_t* __restrict__ deltas) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const DeltaBlock& B = blocks[last_at_or_before<DeltaBlock, &DeltaBlock::start>(blocks, n_blocks, i)];
    uint64_t d = 0;                                // the stream's last value, and values of no stream, add nothing
    if (i >= B.start && i < B.last) {
      const int64_t j = i - B.start;
      const int64_t m = j / (int64_t)B.per_mb;
      const uint8_t* w = chunk + B.widths_off;
      uint64_t bit = 0;
      for (int64_t k = 0; k < m; ++k) bit += (uint64_t)w[k] * B.per_mb;
      const uint32_t bw = w[m];
      bit += (uint64_t)(j - m * (int64_t)B.per_mb) * bw;
      const uint8_t* p = chunk + B.mb_off + (bit >> 3);
      uint64_t lo = 0;
#pragma unroll
      for (int b = 0; b < 8; ++b) lo |= (uint64_t)p[b] << (8 * b);
      const int sh = (int)(bit & 7);
      uint64_t v = lo >> sh;
      if (sh && bw + sh > 64) v |= (uint64_t)p[8] << (64 - sh);        // 64 value bits + 7 bits of offset: a 9-byte window (buffers are padded)
      if (bw < 64) v &= (1ull << bw) - 1;
      d = B.min_delta + v;                         // wrapping: the result is the same whether the writer's deltas were 32- or 64-bit
    }
    deltas[i] = d;
  }
}
// value = the stream's first value + the deltas since; stored as its low `width` (4 or 8) bytes.  Values of no stream are left alone.
__global__ void delta_values_kernel(const DeltaBlock* __restrict__ blocks, int n_blocks, const uint64_t* __restrict__ sums, int64_t n, int width, uint8_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const DeltaBlock& B = blocks[last_at_or_before<DeltaBlock, &DeltaBlock::start>(blocks, n_blocks, i)];
    if (i < B.first || i > B.last) continue;
    const uint64_t v = B.first_value + (sums[i] - sums[B.first]);
    if (width == 8) reinterpret_cast<uint64_t*>(out)[i] = v;
    else reinterpret_cast<uint32_t*>(out)[i] = (uint32_t)v;
  }
}
// BYTE_STREAM_SPLIT: byte b of the page's value k sits at b * count + k
__global__ void byte_stream_split_kernel(const uint8_t* __restrict__ chunk, const DecPage* __restrict__ pages, int n_pages, int64_t n, int width, uint8_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const DecPage& P = pages[last_at_or_before<DecPage, &DecPage::first>(pages, n_pages, i)];
    if (P.encoding != ENC_BSS) continue;
    const uint8_t* src = chunk + P.data_off + (i - P.first);
    for (int b = 0; b < width; ++b) out[i * width + b] = src[(int64_t)b * P.count];
  }
}

struct StringParams {
  const uint8_t* chunk; const DecPage* pages; int n_pages; int64_t n;
  const uint32_t* sfx_len; const uint32_t* pfx_len;   // per decoded value: suffix (or whole-value) length, prefix length (0 but in DELTA_BYTE_ARRAY pages)
  const uint64_t* sfx_pos;                            // exclusive scan of sfx_len
  const uint64_t* pfx_pos;                            // exclusive scan of pfx_len; null for FIXED_LEN_BYTE_ARRAY
  uint8_t* heap;                                      // DELTA_BYTE_ARRAY values: at pfx_pos + sfx_pos, or i * type_length
  ulonglong2* views;                                  // Utf8View output; null for FIXED_LEN_BYTE_ARRAY
  int type_length;                                    // 0 for BYTE_ARRAY
  uint32_t* error;
};
__device__ __forceinline__ uint64_t heap_pos(const StringParams& S, int64_t i) { return S.pfx_pos ? S.pfx_pos[i] + S.sfx_pos[i] : (uint64_t)i * S.type_length; }

__device__ __forceinline__ ulonglong2 make_view(const uint8_t* s, uint32_t len) {
  ulonglong2 v; v.x = len; v.y = 0;
  if (len <= 12) {
    for (uint32_t k = 0; k < len; ++k) { const unsigned long long b = s[k]; if (k < 4) v.x |= b << (32 + 8 * k); else v.y |= b << (8 * (k - 4)); }
  } else {
    for (uint32_t k = 0; k < 4; ++k) v.x |= (unsigned long long)s[k] << (32 + 8 * k);
    v.y = reinterpret_cast<unsigned long long>(s);
  }
  return v;
}
// every value's suffix, checked against its page: DELTA_LENGTH_BYTE_ARRAY values become views into the chunk, DELTA_BYTE_ARRAY
// suffixes are copied to the value's place in the heap (its prefix follows in delta_prefix_kernel)
__global__ void delta_suffix_kernel(StringParams S) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < S.n; i += (int64_t)gridDim.x * blockDim.x) {
    const DecPage& P = S.pages[last_at_or_before<DecPage, &DecPage::first>(S.pages, S.n_pages, i)];
    if (P.encoding != ENC_DLBA && P.encoding != ENC_DBA) continue;
    const uint64_t s = S.sfx_len[i], p = S.pfx_len[i], pos = S.sfx_pos[i] - S.sfx_pos[P.first];
    const bool last = i == P.first + P.count - 1;
    if (s > INT32_MAX || p > INT32_MAX || pos + s > P.data_len || (last && pos + s != P.data_len) || (S.type_length && p + s != (uint64_t)S.type_length)) {
      atomicOr(S.error, ERR_CORRUPT_STREAM);
      continue;
    }
    const uint8_t* src = S.chunk + P.data_off + pos;
    if (P.encoding == ENC_DLBA) { S.views[i] = make_view(src, (uint32_t)s); continue; }
    uint8_t* dst = S.heap + heap_pos(S, i) + p;
    for (uint64_t k = 0; k < s; ++k) dst[k] = src[k];
  }
}
// DELTA_BYTE_ARRAY prefixes, one warp per page (each page starts from an empty previous value): value k's prefix is copied from
// value k-1's bytes once they are complete, then the page's views are built
__global__ void delta_prefix_kernel(StringParams S) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t pg = gw; pg < S.n_pages; pg += nw) {
    const DecPage P = S.pages[pg];
    if (P.encoding != ENC_DBA) continue;
    bool ok = true;
    for (int64_t i = P.first; i < P.first + P.count; ++i) {
      const uint64_t p = S.pfx_len[i];
      const uint64_t prev = i > P.first ? (uint64_t)S.pfx_len[i - 1] + S.sfx_len[i - 1] : 0;
      if (p > prev || (S.type_length && p + S.sfx_len[i] != (uint64_t)S.type_length)) { ok = false; break; }     // checked before anything is read
      const uint8_t* src = S.heap + (p ? heap_pos(S, i - 1) : 0);
      uint8_t* dst = S.heap + heap_pos(S, i);
      for (uint64_t b = lane; b < p; b += 32) dst[b] = src[b];
      __syncwarp();
    }
    if (!ok) { if (lane == 0) atomicOr(S.error, ERR_CORRUPT_STREAM); continue; }
    if (S.views)
      for (int64_t i = P.first + lane; i < P.first + P.count; i += 32) S.views[i] = make_view(S.heap + heap_pos(S, i), S.pfx_len[i] + S.sfx_len[i]);
  }
}

// ---- values -> Arrow ------------------------------------------------------------------------------------
enum { SEG_PLAIN = 0, SEG_DICT = 1, SEG_DECODED = 2 };
// one data page: dense index of its first value, where its values come from (the chunk, the dictionary or the decoded buffer)
// and where they start (byte offset inside the chunk, or inside the decoded buffer)
struct Segment { int64_t dense_start; int64_t byte_off; int64_t kind; };
struct DecodeParams {
  const uint8_t* chunk;
  const uint8_t* decoded;           // values of DELTA / BYTE_STREAM_SPLIT pages in PLAIN layout (views for strings), or null
  const uint32_t* valid;            // per row (1 = value present) or null
  const uint64_t* vpos;             // per row: dense value index (exclusive scan of valid) or null (= row)
  const uint32_t* dict_idx;         // per dense value: dictionary index, or null (PLAIN)
  const uint8_t* dict_vals;         // dictionary in Arrow layout (out_width bytes per entry)
  const Segment* segs; int n_segs;  // data pages
  const uint64_t* str_off;          // PLAIN BYTE_ARRAY: byte offset of every dense value's length prefix inside the chunk
  int64_t n_rows;
  int physical, type_length, out_width;   // out_width: 1 / 2 (narrow integers from INT32), 4, 8, 16 (Decimal128) or 16 with is_view
  int is_view;
  uint32_t dict_size;
  uint32_t* error;
};
__device__ __forceinline__ void store_plain(const DecodeParams& D, const uint8_t* src, uint8_t* dst) {
  if (D.is_view) {
    uint32_t len; memcpy(&len, src, 4);
    *reinterpret_cast<ulonglong2*>(dst) = make_view(src + 4, len);
  } else if (D.physical == PT_FLBA) {           // big-endian two's complement, type_length bytes -> Decimal128
    unsigned __int128 v = (src[0] & 0x80) ? ~(unsigned __int128)0 : 0;
    for (int b = 0; b < D.type_length; ++b) v = (v << 8) | src[b];
    ulonglong2 w; w.x = (unsigned long long)v; w.y = (unsigned long long)(v >> 64);
    *reinterpret_cast<ulonglong2*>(dst) = w;
  } else if (D.physical == PT_INT32 || D.physical == PT_FLOAT) {
    int32_t x; memcpy(&x, src, 4);
    if (D.out_width == 16) { ulonglong2 w; w.x = (unsigned long long)(long long)x; w.y = (unsigned long long)((long long)x >> 63); *reinterpret_cast<ulonglong2*>(dst) = w; }
    else if (D.out_width == 8) *reinterpret_cast<long long*>(dst) = x;
    else if (D.out_width == 4) *reinterpret_cast<int32_t*>(dst) = x;
    else if (D.out_width == 2) *reinterpret_cast<uint16_t*>(dst) = (uint16_t)x;     // Int16 / UInt16: the low bytes of the INT32
    else *dst = (uint8_t)x;                                                         // Int8 / UInt8
  } else {                                      // INT64 / DOUBLE
    long long x; memcpy(&x, src, 8);
    if (D.out_width == 16) { ulonglong2 w; w.x = (unsigned long long)x; w.y = (unsigned long long)(x >> 63); *reinterpret_cast<ulonglong2*>(dst) = w; }
    else *reinterpret_cast<long long*>(dst) = x;
  }
}
__global__ void decode_values_kernel(DecodeParams D, uint8_t* __restrict__ out) {
  const int vw = D.physical == PT_FLBA ? D.type_length : (D.physical == PT_INT32 || D.physical == PT_FLOAT) ? 4 : 8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < D.n_rows; i += (int64_t)gridDim.x * blockDim.x) {
    uint8_t* dst = out + i * D.out_width;
    if (D.valid && !D.valid[i]) {
      if (D.out_width == 16) { ulonglong2 z; z.x = 0; z.y = 0; *reinterpret_cast<ulonglong2*>(dst) = z; }
      else if (D.out_width == 8) *reinterpret_cast<long long*>(dst) = 0;
      else if (D.out_width == 4) *reinterpret_cast<int32_t*>(dst) = 0;
      else if (D.out_width == 2) *reinterpret_cast<uint16_t*>(dst) = 0;
      else *dst = 0;
      continue;
    }
    const int64_t v = D.vpos ? (int64_t)D.vpos[i] : i;
    int lo = 0, hi = D.n_segs - 1;               // the page this value came from
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (D.segs[mid].dense_start <= v) lo = mid; else hi = mid - 1; }
    const Segment& S = D.segs[lo];
    if (S.kind == SEG_DECODED) {                 // PLAIN layout in the decoded buffer; strings are views already
      const uint8_t* src = D.decoded + S.byte_off + (v - S.dense_start) * (D.is_view ? 16 : vw);
      if (D.is_view) *reinterpret_cast<ulonglong2*>(dst) = *reinterpret_cast<const ulonglong2*>(src);
      else store_plain(D, src, dst);
    } else if (S.kind == SEG_DICT) {
      const uint32_t k = D.dict_idx[v];
      if (k >= D.dict_size) { atomicOr(D.error, ERR_UNSUPPORTED); continue; }
      const uint8_t* s = D.dict_vals + (size_t)k * D.out_width;       // entries were decoded at the output width
      if (D.out_width == 16) *reinterpret_cast<ulonglong2*>(dst) = *reinterpret_cast<const ulonglong2*>(s);
      else if (D.out_width == 8) *reinterpret_cast<long long*>(dst) = *reinterpret_cast<const long long*>(s);
      else if (D.out_width == 4) *reinterpret_cast<int32_t*>(dst) = *reinterpret_cast<const int32_t*>(s);
      else if (D.out_width == 2) *reinterpret_cast<uint16_t*>(dst) = *reinterpret_cast<const uint16_t*>(s);
      else *dst = *s;
    } else if (D.is_view) {
      store_plain(D, D.chunk + D.str_off[v], dst);
    } else {
      store_plain(D, D.chunk + S.byte_off + (v - S.dense_start) * vw, dst);
    }
  }
}

BufPtr upload_vec(Ctx* ctx, const void* p, size_t bytes) {
  BufPtr b = dev_alloc(ctx, bytes);
  if (bytes) SG_CUDA(cudaMemcpyAsync(b->ptr, p, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return b;
}

// ---- ZSTD pages -> decompressed image ------------------------------------------------------------------------------------
enum { CODEC_NONE = 0, CODEC_ZSTD = 6 };
// one page of a ZSTD chunk: `copy` bytes (the page header, plus the levels of a data page V2, or the whole body of a V2 page
// stored uncompressed) are copied as they are, then `comp` bytes of frames decompress to exactly `out` bytes
struct ZPage { uint64_t src, dst; uint32_t copy, comp, out, pad; };

constexpr int kZstdWarps = 4;      // warps per block; each warp owns a ZWork in shared memory and kBlockMax bytes of literal scratch

__global__ void __launch_bounds__(kZstdWarps * 32) parquet_zstd_decompress_kernel(const uint8_t* __restrict__ src, const ZPage* __restrict__ pages, int n_pages,
                                                                               uint8_t* __restrict__ image, uint8_t* __restrict__ lits, uint32_t* __restrict__ status) {
  __shared__ zstd::ZWork work[kZstdWarps];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * kZstdWarps + wid, nw = gridDim.x * kZstdWarps;
  const zstd::WarpTeam team{lane};
  uint8_t* my_lits = lits + (size_t)gw * zstd::kBlockMax;
  for (int pg = gw; pg < n_pages; pg += nw) {
    const ZPage P = pages[pg];
    for (uint32_t i = lane; i < P.copy; i += 32) image[P.dst + i] = src[P.src + i];
    int st = zstd::ZS_OK;
    if (P.comp) st = zstd::decode_frames(team, &work[wid], src + P.src + P.copy, P.comp, image + P.dst + P.copy, P.out, my_lits);
    if (lane == 0) status[pg] = (uint32_t)st;
    __syncwarp();
  }
}

std::string zstd_page_name(const Field& f, size_t page) { return "ZSTD page " + std::to_string(page) + " of column '" + f.name + "'"; }
[[noreturn]] void zstd_page_fail(const Field& f, size_t page, int status) {
  if (status == zstd::ZS_UNSUPPORTED) fail(SAILGPU_ERR_UNSUPPORTED, "parquet: " + zstd_page_name(f, page) + " needs a dictionary or holds a skippable frame");
  fail(SAILGPU_ERR_INVALID, "parquet: " + zstd_page_name(f, page) + " is corrupt");
}

}  // namespace

struct ParquetColumnDesc {      // mirrors sailgpu_parquet_column (include/sailgpu.h)
  const uint8_t* chunk; uint64_t chunk_len;
  int32_t physical_type, type_length, max_def_level, codec;
  int64_t num_values;
};

// Everything the host has to find out about a column chunk before the device can decode it: where the pages are, the run
// headers of their level / index streams, how many values each page really carries.  Pure host code (no device touched).
struct ColumnPlan {
  std::vector<Run> level_runs, index_runs;
  std::vector<Segment> segs;
  std::vector<uint64_t> str_off;
  std::vector<std::pair<const uint8_t*, uint64_t>> bodies;     // every page body walked (decompressed for ZSTD), in page order
  int64_t dense = 0, dict_count = 0, dict_len = 0, n_pages = 0;
  const uint8_t* dict_bytes = nullptr;
  bool any_dict_page = false, any_plain_page = false, is_str = false;
  int out_width = 0;
  // DELTA / BYTE_STREAM_SPLIT pages, in decoded space (see DeltaBlock)
  std::vector<DecPage> dec_pages;
  std::vector<DeltaBlock> value_blocks;    // DELTA_BINARY_PACKED values, or the value / suffix lengths of the string encodings
  std::vector<DeltaBlock> prefix_blocks;   // DELTA_BYTE_ARRAY prefix lengths
  int64_t decoded = 0, delta_pages = 0, bss_pages = 0, delta_values = 0, bss_values = 0, dba_pages = 0, dlba_pages = 0;
};

// Walks the DELTA_BINARY_PACKED stream of `count` values at [p, end) of data page `page` into `blocks` (decoded indices from
// `first`); returns where the stream ends.  The header holds the block size, miniblocks per block, the total count and the
// first value; every block holds its min delta, one bit width per miniblock and the miniblocks.  No per-value state is kept.
const uint8_t* walk_delta_stream(const Field& f, int64_t page, const uint8_t* base, const uint8_t* p, const uint8_t* end, int64_t count, int64_t first,
                                 std::vector<DeltaBlock>* blocks) {
  const std::string where = "parquet: DELTA_BINARY_PACKED stream of data page " + std::to_string(page) + " of column '" + f.name + "'";
  auto varint = [&]() -> uint64_t {
    uint64_t v = 0;
    for (int sh = 0;; sh += 7) {
      SG_CHECK(p < end && sh < 64, SAILGPU_ERR_INVALID, where + " overruns its page");
      const uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7F) << sh;
      if (!(b & 0x80)) return v;
    }
  };
  auto zigzag = [&]() -> uint64_t { const uint64_t v = varint(); return (v >> 1) ^ (0 - (v & 1)); };
  const uint64_t block = varint(), n_mb = varint(), total = varint(), first_value = zigzag();
  SG_CHECK(block > 0 && block % 128 == 0 && block <= (1u << 30), SAILGPU_ERR_INVALID, where + ": block size " + std::to_string(block) + " is not a multiple of 128");
  SG_CHECK(n_mb > 0 && block % n_mb == 0 && (block / n_mb) % 32 == 0, SAILGPU_ERR_INVALID,
           where + ": " + std::to_string(n_mb) + " miniblocks per block of " + std::to_string(block) + " values: values per miniblock must be a multiple of 32");
  SG_CHECK(total == (uint64_t)count, SAILGPU_ERR_INVALID, where + " holds " + std::to_string(total) + " values, the page " + std::to_string(count));
  if (count == 0) return p;
  const uint64_t per_mb = block / n_mb;
  const int64_t last = first + count - 1;
  DeltaBlock B{first, first, last, first_value, 0, 0, 0, per_mb};
  if (count == 1) { blocks->push_back(B); return p; }       // no block follows: the first value is the stream
  for (int64_t left = count - 1; left > 0; left -= std::min<int64_t>(left, (int64_t)block), B.start += (int64_t)block) {
    B.min_delta = zigzag();
    SG_CHECK((uint64_t)(end - p) >= n_mb, SAILGPU_ERR_INVALID, where + " overruns its page");
    B.widths_off = (uint64_t)(p - base);
    const uint64_t used = std::min<uint64_t>(n_mb, ((uint64_t)left + per_mb - 1) / per_mb);   // the last block's unused miniblocks have no bodies
    uint64_t body = 0;
    for (uint64_t m = 0; m < used; ++m) {
      SG_CHECK(p[m] <= 64, SAILGPU_ERR_INVALID, where + ": bit width " + std::to_string(p[m]));
      body += p[m] * per_mb / 8;
    }
    p += n_mb;
    B.mb_off = (uint64_t)(p - base);
    SG_CHECK((uint64_t)(end - p) >= body, SAILGPU_ERR_INVALID, where + " overruns its page");
    p += body;
    blocks->push_back(B);
  }
  return p;
}

void check_parquet_column(const Field& f, const ParquetColumnDesc& c, int64_t n_rows) {
  SG_CHECK(c.codec == CODEC_NONE || c.codec == CODEC_ZSTD, SAILGPU_ERR_UNSUPPORTED,
           "parquet: only uncompressed and ZSTD pages are decoded on the GPU path (column '" + f.name + "' has codec " + std::to_string(c.codec) + ")");
  SG_CHECK(c.max_def_level == 0 || c.max_def_level == 1, SAILGPU_ERR_UNSUPPORTED, "parquet: nested / repeated columns are not supported (column '" + f.name + "')");
  SG_CHECK(c.num_values == n_rows, SAILGPU_ERR_INVALID, "parquet: column '" + f.name + "' has " + std::to_string(c.num_values) + " values for " + std::to_string(n_rows) + " rows");
  const int pt = c.physical_type;
  const bool is_str = f.type.is_string();
  SG_CHECK(pt == PT_INT32 || pt == PT_INT64 || pt == PT_DOUBLE || pt == PT_FLBA || pt == PT_BYTE_ARRAY, SAILGPU_ERR_UNSUPPORTED,
           "parquet: physical type " + std::to_string(pt) + " (column '" + f.name + "')");
  SG_CHECK((pt == PT_BYTE_ARRAY) == is_str, SAILGPU_ERR_UNSUPPORTED, "parquet: BYTE_ARRAY columns decode to strings only (column '" + f.name + "')");
  SG_CHECK(f.type.id != TypeId::Utf8, SAILGPU_ERR_UNSUPPORTED, "parquet: strings decode to Utf8View (what Sail reads Parquet strings as: application.yaml:375-381)");
  const int out_width = is_str ? 16 : f.type.arrow_width();
  const bool narrow = f.type.is_int() && out_width <= 2;                      // Int8 / Int16 / UInt8 / UInt16
  SG_CHECK(narrow || out_width == 4 || out_width == 8 || out_width == 16, SAILGPU_ERR_UNSUPPORTED, "parquet: target type " + f.type.str());
  if (pt == PT_FLBA) SG_CHECK(f.type.is_decimal() && c.type_length >= 1 && c.type_length <= 16, SAILGPU_ERR_UNSUPPORTED, "parquet: FIXED_LEN_BYTE_ARRAY decodes to Decimal128 only");
  if (pt == PT_DOUBLE) SG_CHECK(f.type.id == TypeId::Float64, SAILGPU_ERR_UNSUPPORTED, "parquet: DOUBLE decodes to Float64");
  if (pt == PT_INT32) SG_CHECK(narrow || out_width == 4 || f.type.is_decimal(), SAILGPU_ERR_UNSUPPORTED, "parquet: INT32 decodes to 8-, 16- or 32-bit types or Decimal128");
  if (pt == PT_INT64) SG_CHECK(out_width == 8 || f.type.is_decimal(), SAILGPU_ERR_UNSUPPORTED, "parquet: INT64 decodes to 64-bit types or Decimal128");
}

// Walks the page headers of a ZSTD chunk into `pages` (source offsets from src_base, image offsets from dst_base) and checks
// the first frame header of every page: magic number, no dictionary, a content size that fits the page.  Stops where
// plan_parquet_column stops, once the data pages hold n_rows values.  Returns the length of the chunk's image.
uint64_t plan_zstd_pages(const Field& f, const ParquetColumnDesc& c, int64_t n_rows, uint64_t src_base, uint64_t dst_base, std::vector<ZPage>* pages) {
  const uint8_t* end = c.chunk + c.chunk_len;
  TReader r{c.chunk, end};
  uint64_t dst = dst_base;
  int64_t rows_done = 0;
  for (size_t idx = 0; r.p < end && rows_done < n_rows; ++idx) {
    const uint8_t* start = r.p;
    const PageHeader h = read_page_header(r);
    SG_CHECK(h.compressed >= 0 && h.uncompressed >= 0 && r.p + h.compressed <= end, SAILGPU_ERR_INVALID, "parquet: page overruns its column chunk");
    uint32_t keep = 0;                           // body bytes stored uncompressed
    if (h.type == PAGE_DATA_V2) {
      SG_CHECK(h.def_bytes >= 0 && h.rep_bytes >= 0, SAILGPU_ERR_INVALID, "parquet: negative level length");
      keep = h.v2_compressed ? (uint32_t)h.def_bytes + (uint32_t)h.rep_bytes : (uint32_t)h.compressed;
      SG_CHECK(h.v2_compressed || h.compressed == h.uncompressed, SAILGPU_ERR_INVALID, "parquet: uncompressed page V2 with two sizes");
      SG_CHECK(keep <= (uint32_t)h.compressed && keep <= (uint32_t)h.uncompressed, SAILGPU_ERR_INVALID, "parquet: levels overrun their page");
    }
    const uint32_t hdr = (uint32_t)(r.p - start);
    const ZPage p{src_base + (uint64_t)(start - c.chunk), dst, hdr + keep, (uint32_t)h.compressed - keep, (uint32_t)h.uncompressed - keep, 0};
    if (p.comp) {
      zstd::FrameHeader fh;
      const int st = zstd::parse_frame_header(start + p.copy, p.comp, &fh);
      if (st) zstd_page_fail(f, idx, st);
      if (fh.has_content_size && fh.content_size > p.out) zstd_page_fail(f, idx, zstd::ZS_CORRUPT);
    } else if (p.out) zstd_page_fail(f, idx, zstd::ZS_CORRUPT);
    pages->push_back(p);
    dst += (uint64_t)p.copy + p.out;
    r.p += h.compressed;
    if (h.type == PAGE_DATA || h.type == PAGE_DATA_V2) rows_done += h.num_values;
  }
  return dst - dst_base;
}

// The decompressed image of a ZSTD chunk, built on the host by the same decoder (sailgpu_parquet_inspect)
std::vector<uint8_t> zstd_image_host(const Field& f, const ParquetColumnDesc& c, int64_t n_rows, uint64_t* image_len) {
  std::vector<ZPage> pages;
  *image_len = plan_zstd_pages(f, c, n_rows, 0, 0, &pages);
  std::vector<uint8_t> img(*image_len + 64, 0), lits(zstd::kBlockMax);
  auto work = std::make_unique<zstd::ZWork>();
  for (size_t i = 0; i < pages.size(); ++i) {
    const ZPage& p = pages[i];
    memcpy(img.data() + p.dst, c.chunk + p.src, p.copy);
    if (!p.comp) continue;
    const int st = zstd::decode_frames(zstd::SerialTeam{}, work.get(), c.chunk + p.src + p.copy, p.comp, img.data() + p.dst + p.copy, p.out, lits.data());
    if (st) zstd_page_fail(f, i, st);
  }
  return img;
}

// `c` describes the chunk as stored when it is uncompressed, and its decompressed image when its codec is ZSTD
ColumnPlan plan_parquet_column(const Field& f, const ParquetColumnDesc& c, int64_t n_rows) {
  ColumnPlan P;
  check_parquet_column(f, c, n_rows);
  const bool is_str = f.type.is_string();
  P.is_str = is_str;
  P.out_width = is_str ? 16 : f.type.arrow_width();
  const bool image = c.codec == CODEC_ZSTD;

  // ---- host: page headers and run headers -----------------------------------------------------------------------
  const uint8_t* base = c.chunk; const uint8_t* end = c.chunk + c.chunk_len;
  std::vector<Run>& level_runs = P.level_runs; std::vector<Run>& index_runs = P.index_runs;
  std::vector<Segment>& segs = P.segs;
  std::vector<uint64_t>& str_off = P.str_off;
  int64_t rows_done = 0; int64_t& dense_done = P.dense;
  bool have_dict = false; bool& any_dict_page = P.any_dict_page; bool& any_plain_page = P.any_plain_page;
  int64_t& dict_count = P.dict_count; const uint8_t*& dict_bytes = P.dict_bytes; int64_t& dict_len = P.dict_len;
  TReader r{base, end};
  while (r.p < end && rows_done < n_rows) {
    const PageHeader h = read_page_header(r);
    if (!image) SG_CHECK(h.compressed == h.uncompressed, SAILGPU_ERR_UNSUPPORTED, "parquet: compressed page in column '" + f.name + "'");
    const int64_t body_len = image ? h.uncompressed : h.compressed;      // an image holds every body decompressed
    SG_CHECK(body_len >= 0, SAILGPU_ERR_INVALID, "parquet: negative page size");
    const uint8_t* body = r.p; const uint8_t* body_end = body + body_len;
    SG_CHECK(body_end <= end, SAILGPU_ERR_INVALID, "parquet: page overruns its column chunk");
    r.p = body_end;
    P.bodies.emplace_back(body, (uint64_t)body_len);
    if (h.type == PAGE_DICT) {
      SG_CHECK(h.encoding == ENC_PLAIN || h.encoding == ENC_PLAIN_DICT, SAILGPU_ERR_UNSUPPORTED, "parquet: dictionary page encoding " + std::to_string(h.encoding));
      have_dict = true; dict_count = h.num_values; dict_bytes = body; dict_len = body_len;
      continue;
    }
    if (h.type != PAGE_DATA && h.type != PAGE_DATA_V2) continue;       // index pages etc.
    P.n_pages++;
    const int64_t nv = h.num_values;
    const uint8_t* vals = body;
    int64_t non_null = nv;
    if (h.type == PAGE_DATA_V2) {
      SG_CHECK(h.rep_bytes == 0, SAILGPU_ERR_UNSUPPORTED, "parquet: repetition levels");
      if (c.max_def_level > 0) non_null = scan_hybrid(base, body, body + h.def_bytes, 1, nv, rows_done, &level_runs, 1);
      vals = body + h.def_bytes;
    } else if (c.max_def_level > 0) {
      SG_CHECK(h.def_encoding == ENC_RLE, SAILGPU_ERR_UNSUPPORTED, "parquet: definition levels must be RLE encoded");
      uint32_t len; memcpy(&len, body, 4);
      SG_CHECK(body + 4 + len <= body_end, SAILGPU_ERR_INVALID, "parquet: definition levels overrun their page");
      non_null = scan_hybrid(base, body + 4, body + 4 + len, 1, nv, rows_done, &level_runs, 1);
      vals = body + 4 + len;
    }
    if (h.encoding == ENC_RLE_DICT || h.encoding == ENC_PLAIN_DICT) {
      SG_CHECK(have_dict, SAILGPU_ERR_INVALID, "parquet: dictionary-encoded page without a dictionary page");
      any_dict_page = true;
      segs.push_back(Segment{dense_done, 0, SEG_DICT});
      SG_CHECK(vals < body_end || non_null == 0, SAILGPU_ERR_INVALID, "parquet: empty dictionary-index stream");
      if (non_null > 0) {
        const int bw = vals[0];
        SG_CHECK(bw <= 32, SAILGPU_ERR_INVALID, "parquet: dictionary index width " + std::to_string(bw));
        if (bw == 0) index_runs.push_back(Run{dense_done, 0, (uint32_t)non_null, 0, 0, 0});
        else scan_hybrid(base, vals + 1, body_end, bw, non_null, dense_done, &index_runs, 0xFFFFFFFFu);
      }
    } else if (h.encoding == ENC_PLAIN) {
      any_plain_page = true;
      segs.push_back(Segment{dense_done, (int64_t)(vals - base), SEG_PLAIN});
      if (is_str) {
        // offsets are indexed by dense value number: values of earlier DICTIONARY pages get a zero (never read) -- filled
        // only now, so that an all-dictionary chunk keeps no per-value host state at all
        str_off.resize((size_t)dense_done, 0);
        const uint8_t* q = vals;
        for (int64_t i = 0; i < non_null; ++i) {
          SG_CHECK(q + 4 <= body_end, SAILGPU_ERR_INVALID, "parquet: BYTE_ARRAY value overruns its page");
          uint32_t len; memcpy(&len, q, 4);
          str_off.push_back((uint64_t)(q - base));
          q += 4 + (size_t)len;
        }
        SG_CHECK(q <= body_end, SAILGPU_ERR_INVALID, "parquet: BYTE_ARRAY value overruns its page");
      }
    } else if (h.encoding == ENC_DBP || h.encoding == ENC_DLBA || h.encoding == ENC_DBA || h.encoding == ENC_BSS) {
      const int pt = c.physical_type;
      const bool ok = h.encoding == ENC_DBP ? (pt == PT_INT32 || pt == PT_INT64)
                    : h.encoding == ENC_DLBA ? pt == PT_BYTE_ARRAY
                    : h.encoding == ENC_DBA ? (pt == PT_BYTE_ARRAY || pt == PT_FLBA)
                    : (pt == PT_INT32 || pt == PT_INT64 || pt == PT_DOUBLE || pt == PT_FLBA);
      SG_CHECK(ok, SAILGPU_ERR_UNSUPPORTED, "parquet: value encoding " + std::to_string(h.encoding) + " for physical type " + std::to_string(pt) + " (column '" + f.name + "')");
      const int64_t page = P.n_pages - 1;
      const std::string where = "parquet: data page " + std::to_string(page) + " of column '" + f.name + "'";
      const int vw = pt == PT_FLBA ? c.type_length : pt == PT_INT32 ? 4 : 8;
      segs.push_back(Segment{dense_done, P.decoded * (is_str ? 16 : vw), SEG_DECODED});
      DecPage dp{P.decoded, non_null, 0, 0, h.encoding};
      if (h.encoding == ENC_BSS) {
        SG_CHECK(body_end - vals == non_null * vw, SAILGPU_ERR_INVALID, where + ": BYTE_STREAM_SPLIT values do not fill the page");
        dp.data_off = (uint64_t)(vals - base); dp.data_len = (uint64_t)(body_end - vals);
        P.bss_pages++; P.bss_values += non_null;
      } else {
        const uint8_t* q = vals;
        if (h.encoding == ENC_DBA) q = walk_delta_stream(f, page, base, q, body_end, non_null, P.decoded, &P.prefix_blocks);
        q = walk_delta_stream(f, page, base, q, body_end, non_null, P.decoded, &P.value_blocks);
        if (h.encoding == ENC_DBP) SG_CHECK(q == body_end, SAILGPU_ERR_INVALID, where + ": the DELTA_BINARY_PACKED stream ends " + std::to_string(body_end - q) + " bytes before the page");
        dp.data_off = (uint64_t)(q - base); dp.data_len = (uint64_t)(body_end - q);   // the string bytes; the device checks the lengths add up to them
        P.delta_pages++; P.delta_values += non_null;
        P.dba_pages += h.encoding == ENC_DBA; P.dlba_pages += h.encoding == ENC_DLBA;
      }
      P.dec_pages.push_back(dp);
      P.decoded += non_null;
    } else fail(SAILGPU_ERR_UNSUPPORTED, "parquet: value encoding " + std::to_string(h.encoding) + " (column '" + f.name + "')");
    rows_done += nv; dense_done += non_null;
  }
  SG_CHECK(rows_done == n_rows, SAILGPU_ERR_INVALID, "parquet: pages of column '" + f.name + "' hold " + std::to_string(rows_done) + " values, expected " + std::to_string(n_rows));
  // (a writer that outgrows its dictionary falls back to PLAIN pages mid-chunk: every page carries its own kind)

  return P;
}

// The values of a column's DELTA / BYTE_STREAM_SPLIT pages, decoded into one buffer in PLAIN layout (16-byte views for strings).
// A DELTA_BYTE_ARRAY string column also gets a heap holding its rebuilt values, which its views point into.
BufPtr decode_delta_pages(Ctx* ctx, const ColumnPlan& P, const ParquetColumnDesc& c, const uint8_t* dbase, uint32_t* error, BufPtr* heap) {
  const int64_t n = P.decoded;
  const int pt = c.physical_type;
  const bool lengths = P.is_str || pt == PT_FLBA;     // the DELTA streams hold string lengths, not values
  const int vw = P.is_str ? 16 : pt == PT_FLBA ? c.type_length : pt == PT_INT32 ? 4 : 8;
  const int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  BufPtr out = dev_alloc(ctx, (size_t)n * vw + 64);
  BufPtr dpages = upload_vec(ctx, P.dec_pages.data(), P.dec_pages.size() * sizeof(DecPage));
  const DecPage* pages = static_cast<const DecPage*>(dpages->ptr);
  BufPtr scan_scratch = dev_alloc(ctx, 1026 * 8);
  // DELTA_BINARY_PACKED: one thread per value unpacks its delta, a wrapping 64-bit scan adds them up
  auto unpack = [&](const std::vector<DeltaBlock>& blocks, int width, void* dst) {
    if (blocks.empty()) return;
    BufPtr dblocks = upload_vec(ctx, blocks.data(), blocks.size() * sizeof(DeltaBlock));
    BufPtr deltas = dev_alloc(ctx, (size_t)n * 8), sums = dev_alloc(ctx, (size_t)n * 8);
    const DeltaBlock* b = static_cast<const DeltaBlock*>(dblocks->ptr);
    delta_unpack_kernel<<<grid, 256, 0, ctx->stream>>>(dbase, b, (int)blocks.size(), n, static_cast<uint64_t*>(deltas->ptr));
    SG_CUDA(cudaGetLastError());
    SG_CUDA(launch_exclusive_scan_u64(static_cast<const uint64_t*>(deltas->ptr), n, static_cast<uint64_t*>(sums->ptr), static_cast<uint64_t*>(scan_scratch->ptr), ctx->stream));
    delta_values_kernel<<<grid, 256, 0, ctx->stream>>>(b, (int)blocks.size(), static_cast<const uint64_t*>(sums->ptr), n, width, static_cast<uint8_t*>(dst));
    SG_CUDA(cudaGetLastError());
  };
  if (P.bss_pages) {
    byte_stream_split_kernel<<<grid, 256, 0, ctx->stream>>>(dbase, pages, (int)P.dec_pages.size(), n, vw, static_cast<uint8_t*>(out->ptr));
    SG_CUDA(cudaGetLastError());
  }
  if (!lengths) { unpack(P.value_blocks, vw, out->ptr); return out; }
  if (!P.dba_pages && !P.dlba_pages) return out;
  // strings: lengths of n values plus a zero, so that the exclusive scans end with their totals
  BufPtr sfx_len = dev_alloc_zero(ctx, (size_t)(n + 1) * 4), pfx_len = dev_alloc_zero(ctx, (size_t)(n + 1) * 4);
  BufPtr sfx_pos = dev_alloc(ctx, (size_t)(n + 1) * 8), pfx_pos;
  unpack(P.value_blocks, 4, sfx_len->ptr);
  unpack(P.prefix_blocks, 4, pfx_len->ptr);
  StringParams S; memset(&S, 0, sizeof(S));
  S.chunk = dbase; S.pages = pages; S.n_pages = (int)P.dec_pages.size(); S.n = n;
  S.sfx_len = static_cast<const uint32_t*>(sfx_len->ptr); S.pfx_len = static_cast<const uint32_t*>(pfx_len->ptr);
  S.sfx_pos = static_cast<const uint64_t*>(sfx_pos->ptr); S.error = error;
  SG_CUDA(launch_exclusive_scan_u32(S.sfx_len, n + 1, static_cast<uint64_t*>(sfx_pos->ptr), static_cast<uint64_t*>(scan_scratch->ptr), ctx->stream));
  if (P.is_str) {
    S.views = static_cast<ulonglong2*>(out->ptr);
    if (P.dba_pages) {                             // the heap: a scan of prefix + suffix lengths, one read-back for its size
      pfx_pos = dev_alloc(ctx, (size_t)(n + 1) * 8);
      SG_CUDA(launch_exclusive_scan_u32(S.pfx_len, n + 1, static_cast<uint64_t*>(pfx_pos->ptr), static_cast<uint64_t*>(scan_scratch->ptr), ctx->stream));
      uint64_t tot[2] = {0, 0};
      SG_CUDA(cudaMemcpyAsync(&tot[0], static_cast<uint64_t*>(pfx_pos->ptr) + n, 8, cudaMemcpyDeviceToHost, ctx->stream));
      SG_CUDA(cudaMemcpyAsync(&tot[1], static_cast<uint64_t*>(sfx_pos->ptr) + n, 8, cudaMemcpyDeviceToHost, ctx->stream));
      stream_sync(ctx);
      SG_CHECK(tot[0] + tot[1] < (1ull << 40), SAILGPU_ERR_INVALID, "parquet: DELTA_BYTE_ARRAY lengths of a column add up to " + std::to_string(tot[0] + tot[1]) + " bytes");
      *heap = dev_alloc(ctx, (size_t)(tot[0] + tot[1]) + 64);
      S.heap = static_cast<uint8_t*>((*heap)->ptr);
      S.pfx_pos = static_cast<const uint64_t*>(pfx_pos->ptr);
    }
  } else {                                         // FIXED_LEN_BYTE_ARRAY: every value is type_length bytes, rebuilt in place
    S.heap = static_cast<uint8_t*>(out->ptr);
    S.type_length = c.type_length;
  }
  delta_suffix_kernel<<<grid, 256, 0, ctx->stream>>>(S);
  SG_CUDA(cudaGetLastError());
  if (P.dba_pages) {
    const int blocks = (int)std::min<int64_t>(((int64_t)P.dec_pages.size() + 7) / 8, grid_cap(8));
    delta_prefix_kernel<<<blocks, 256, 0, ctx->stream>>>(S);
    SG_CUDA(cudaGetLastError());
  }
  return out;               // (scratch buffers go back to the stream-ordered pool; the caller syncs before P's host vectors go)
}

// dimage: for a ZSTD chunk, its image in HBM (c describes the host copy of that image); `image_buf` holds it
DevColumn decode_parquet_column(Ctx* ctx, const Field& f, const ParquetColumnDesc& c, int64_t n_rows, const uint8_t* dimage = nullptr, BufPtr image_buf = nullptr) {
  ColumnPlan P = plan_parquet_column(f, c, n_rows);
  const uint8_t* base = c.chunk;
  const int pt = c.physical_type;
  const bool is_str = P.is_str;
  const int out_width = P.out_width;
  std::vector<Run>& level_runs = P.level_runs; std::vector<Run>& index_runs = P.index_runs;
  std::vector<Segment>& segs = P.segs;
  std::vector<uint64_t>& str_off = P.str_off;
  const int64_t dense_done = P.dense, dict_count = P.dict_count, dict_len = P.dict_len;
  const uint8_t* dict_bytes = P.dict_bytes;
  const bool any_dict_page = P.any_dict_page, any_plain_page = P.any_plain_page;
  // ---- device ---------------------------------------------------------------------------------------------------------
  DevColumn col; col.type = f.type; col.length = n_rows;
  BufPtr dchunk = image_buf;
  if (!dimage) {
    dchunk = dev_alloc(ctx, (size_t)c.chunk_len + 64);
    HostStager st(ctx);
    st.add_raw(dchunk->ptr, c.chunk, (size_t)c.chunk_len);
    st.flush();
  }
  const uint8_t* dbase = dimage ? dimage : static_cast<const uint8_t*>(dchunk->ptr);
  BufPtr err = dev_alloc_zero(ctx, 8);
  auto expand = [&](const std::vector<Run>& runs, int64_t n) -> BufPtr {
    BufPtr out = dev_alloc(ctx, (size_t)n * 4 + 16);
    if (n == 0) return out;
    std::vector<int64_t> starts(runs.size());
    for (size_t i = 0; i < runs.size(); ++i) starts[i] = runs[i].out_start;
    BufPtr druns = upload_vec(ctx, runs.data(), runs.size() * sizeof(Run)), dstarts = upload_vec(ctx, starts.data(), starts.size() * 8);
    expand_runs_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, ctx->stream>>>(dbase, static_cast<const Run*>(druns->ptr), static_cast<const int64_t*>(dstarts->ptr),
                                                                                                (int)runs.size(), n, static_cast<uint32_t*>(out->ptr));
    SG_CUDA(cudaGetLastError());
    stream_sync(ctx);      // `starts` / `runs` are host vectors
    return out;
  };
  DecodeParams D; memset(&D, 0, sizeof(D));
  D.chunk = dbase; D.n_rows = n_rows; D.physical = pt; D.type_length = c.type_length; D.out_width = out_width; D.is_view = is_str ? 1 : 0;
  D.error = static_cast<uint32_t*>(err->ptr);
  BufPtr valid, vpos, scratch, didx, ddict, dsegs, dstr;
  if (c.max_def_level > 0) {
    valid = expand(level_runs, n_rows);
    vpos = dev_alloc(ctx, (size_t)(n_rows + 1) * 8);
    scratch = dev_alloc(ctx, 1026 * 8);
    SG_CUDA(launch_exclusive_scan_u32(static_cast<const uint32_t*>(valid->ptr), n_rows, static_cast<uint64_t*>(vpos->ptr), static_cast<uint64_t*>(scratch->ptr), ctx->stream));
    D.valid = static_cast<const uint32_t*>(valid->ptr); D.vpos = static_cast<const uint64_t*>(vpos->ptr);
  }
  if (any_dict_page) {
    // the dictionary itself is a PLAIN page: decode it into the Arrow layout with the same kernel
    DecodeParams Q; memset(&Q, 0, sizeof(Q));
    Q.chunk = dbase; Q.n_rows = dict_count; Q.physical = pt; Q.type_length = c.type_length; Q.out_width = out_width; Q.is_view = D.is_view; Q.error = D.error;
    std::vector<Segment> ds{Segment{0, (int64_t)(dict_bytes - base), 0}};
    std::vector<uint64_t> doff;
    BufPtr qsegs, qoff;
    if (is_str) {
      const uint8_t* q = dict_bytes;
      for (int64_t i = 0; i < dict_count; ++i) {
        SG_CHECK(q + 4 <= dict_bytes + dict_len, SAILGPU_ERR_INVALID, "parquet: dictionary value overruns its page");
        uint32_t len; memcpy(&len, q, 4);
        doff.push_back((uint64_t)(q - base));
        q += 4 + (size_t)len;
      }
      qoff = upload_vec(ctx, doff.data(), doff.size() * 8);
      Q.str_off = static_cast<const uint64_t*>(qoff->ptr);
    }
    qsegs = upload_vec(ctx, ds.data(), sizeof(Segment));
    Q.segs = static_cast<const Segment*>(qsegs->ptr); Q.n_segs = 1;
    ddict = dev_alloc(ctx, (size_t)std::max<int64_t>(dict_count, 1) * out_width);
    if (dict_count) decode_values_kernel<<<(int)std::min<int64_t>((dict_count + 255) / 256, grid_cap(4)), 256, 0, ctx->stream>>>(Q, static_cast<uint8_t*>(ddict->ptr));
    SG_CUDA(cudaGetLastError());
    stream_sync(ctx);
    didx = expand(index_runs, dense_done);
    D.dict_idx = static_cast<const uint32_t*>(didx->ptr); D.dict_vals = static_cast<const uint8_t*>(ddict->ptr); D.dict_size = (uint32_t)dict_count;
  }
  BufPtr decoded, heap;
  if (P.decoded) decoded = decode_delta_pages(ctx, P, c, dbase, D.error, &heap);
  D.decoded = decoded ? static_cast<const uint8_t*>(decoded->ptr) : nullptr;
  if (is_str && any_plain_page) {
    str_off.resize((size_t)dense_done, 0);
    dstr = upload_vec(ctx, str_off.data(), str_off.size() * 8);
    D.str_off = static_cast<const uint64_t*>(dstr->ptr);
  }
  if (segs.empty()) segs.push_back(Segment{0, 0, 0});
  dsegs = upload_vec(ctx, segs.data(), segs.size() * sizeof(Segment));
  D.segs = static_cast<const Segment*>(dsegs->ptr); D.n_segs = (int)segs.size();
  col.data = dev_alloc(ctx, (size_t)n_rows * out_width);
  if (n_rows) decode_values_kernel<<<(int)std::min<int64_t>((n_rows + 255) / 256, grid_cap(8)), 256, 0, ctx->stream>>>(D, static_cast<uint8_t*>(col.data->ptr));
  SG_CUDA(cudaGetLastError());
  if (is_str) col.heaps = {dchunk};                 // long views point into the chunk bytes
  if (is_str && heap) col.heaps.push_back(heap);    // ... or into the values DELTA_BYTE_ARRAY pages rebuilt
  col.null_count = 0;
  if (c.max_def_level > 0 && dense_done < n_rows) {
    // validity bitmap from the expanded levels (u32 0/1 -> bytes -> bits)
    BufPtr bytes = dev_alloc(ctx, (size_t)n_rows + 4);
    SG_CUDA(launch_u32_to_bytes(static_cast<const uint32_t*>(valid->ptr), static_cast<uint8_t*>(bytes->ptr), n_rows, ctx->stream));
    col.validity = dev_alloc_zero(ctx, (size_t)((n_rows + 31) / 32 * 4));
    SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(bytes->ptr), static_cast<uint32_t*>(col.validity->ptr), n_rows, nullptr, ctx->stream));
    col.null_count = n_rows - dense_done;
  }
  uint32_t e = 0;
  SG_CUDA(cudaMemcpyAsync(&e, err->ptr, 4, cudaMemcpyDeviceToHost, ctx->stream));
  stream_sync(ctx);       // host vectors above; error flag
  SG_CHECK(!(e & ERR_CORRUPT_STREAM), SAILGPU_ERR_INVALID,
           "parquet: corrupt DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY values in column '" + f.name + "' (a length overruns its page or differs from the type length, or a prefix is longer than the value before it)");
  SG_CHECK(e == 0, SAILGPU_ERR_INVALID, "parquet: dictionary index out of range in column '" + f.name + "'");
  return col;
}

// One row group: the compressed pages of every ZSTD column go through one decompression launch and one read-back, then each
// column is decoded (a ZSTD column from its image, an uncompressed one as stored).
void decode_parquet_row_group(Ctx* ctx, const Schema& schema, const std::vector<ParquetColumnDesc>& cols, int64_t n_rows, DevBatch* b) {
  const size_t nc = cols.size();
  std::vector<ZPage> pages;
  std::vector<size_t> first_page(nc + 1, 0);
  std::vector<uint64_t> src_off(nc, 0), img_off(nc, 0), img_len(nc, 0);
  uint64_t src_total = 0, img_total = 0, out_bytes = 0;
  for (size_t i = 0; i < nc; ++i) {
    first_page[i] = pages.size();
    check_parquet_column(schema[i], cols[i], n_rows);
    if (cols[i].codec != CODEC_ZSTD) continue;
    src_off[i] = src_total; img_off[i] = img_total;
    img_len[i] = plan_zstd_pages(schema[i], cols[i], n_rows, src_total, img_total, &pages);
    src_total += cols[i].chunk_len;
    img_total = (img_total + img_len[i] + 63) & ~(uint64_t)63;
  }
  first_page[nc] = pages.size();
  for (const ZPage& p : pages) out_bytes += p.out;
  ctx->parquet_zstd = Ctx::ParquetZstd{};
  BufPtr dimg;
  std::vector<uint8_t> himg;
  const size_t status_bytes = (pages.size() * 4 + 255) & ~(size_t)255;     // per-page status ahead of the images
  bool any_zstd = false;
  for (const ParquetColumnDesc& c : cols) any_zstd |= c.codec == CODEC_ZSTD;
  if (any_zstd) {                                // (a chunk of an empty row group has no page to decompress, but still an image)
    dimg = dev_alloc(ctx, status_bytes + (size_t)img_total + 64);
    himg.assign(status_bytes + (size_t)img_total + 64, 0);
  }
  if (!pages.empty()) {
    SG_CHECK(pages.size() < (size_t)INT32_MAX, SAILGPU_ERR_UNSUPPORTED, "parquet: too many pages in one call");
    BufPtr dsrc = dev_alloc(ctx, (size_t)src_total + 64);
    {
      HostStager st(ctx);
      for (size_t i = 0; i < nc; ++i)
        if (cols[i].codec == CODEC_ZSTD && cols[i].chunk_len) st.add_raw(static_cast<uint8_t*>(dsrc->ptr) + src_off[i], cols[i].chunk, (size_t)cols[i].chunk_len);
      st.flush();
    }
    BufPtr dpages = upload_vec(ctx, pages.data(), pages.size() * sizeof(ZPage));
    int per_sm = 0;
    SG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, parquet_zstd_decompress_kernel, kZstdWarps * 32, 0));
    const int blocks = (int)std::min<int64_t>(((int64_t)pages.size() + kZstdWarps - 1) / kZstdWarps, (int64_t)std::max(per_sm, 1) * ctx->sm_count);
    BufPtr lits = dev_alloc(ctx, (size_t)blocks * kZstdWarps * zstd::kBlockMax);
    uint8_t* dbase = static_cast<uint8_t*>(dimg->ptr);
    cudaEvent_t ev[3];
    for (auto& e : ev) SG_CUDA(cudaEventCreate(&e));
    SG_CUDA(cudaEventRecord(ev[0], ctx->stream));
    parquet_zstd_decompress_kernel<<<blocks, kZstdWarps * 32, 0, ctx->stream>>>(static_cast<const uint8_t*>(dsrc->ptr), static_cast<const ZPage*>(dpages->ptr), (int)pages.size(),
                                                                            dbase + status_bytes, static_cast<uint8_t*>(lits->ptr), reinterpret_cast<uint32_t*>(dbase));
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaEventRecord(ev[1], ctx->stream));
    SG_CUDA(cudaMemcpyAsync(himg.data(), dbase, status_bytes + (size_t)img_total, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaEventRecord(ev[2], ctx->stream));
    stream_sync(ctx);        // the run-header walk reads the images on the host
    ctx->d2h_bytes += status_bytes + img_total;
    Ctx::ParquetZstd& s = ctx->parquet_zstd;
    s.pages = pages.size(); s.out_bytes = out_bytes; s.image_bytes = img_total;
    SG_CUDA(cudaEventElapsedTime(&s.decompress_ms, ev[0], ev[1]));
    SG_CUDA(cudaEventElapsedTime(&s.readback_ms, ev[1], ev[2]));
    for (auto& e : ev) cudaEventDestroy(e);
    const uint32_t* status = reinterpret_cast<const uint32_t*>(himg.data());
    for (size_t i = 0; i < nc; ++i)
      for (size_t k = first_page[i]; k < first_page[i + 1]; ++k)
        if (status[k]) zstd_page_fail(schema[i], k - first_page[i], (int)status[k]);
  }
  for (size_t i = 0; i < nc; ++i) {
    if (cols[i].codec != CODEC_ZSTD) { b->cols.push_back(decode_parquet_column(ctx, schema[i], cols[i], n_rows)); continue; }
    ParquetColumnDesc d = cols[i];
    d.chunk = himg.data() + status_bytes + img_off[i]; d.chunk_len = img_len[i];
    b->cols.push_back(decode_parquet_column(ctx, schema[i], d, n_rows, static_cast<const uint8_t*>(dimg->ptr) + status_bytes + img_off[i], dimg));
  }
}

// FNV-1a, 64 bits
static uint64_t fnv1a(uint64_t h, const uint8_t* p, uint64_t n) {
  for (uint64_t i = 0; i < n; ++i) { h ^= p[i]; h *= 0x100000001b3ull; }
  return h;
}

// host-only summary of a column plan (tests/test_parquet_plan.py pins the page / run walking against pyarrow's own metadata);
// a ZSTD chunk is decompressed on the host by the decoder the device runs
std::string parquet_plan_summary(const Field& f, const ParquetColumnDesc& c, int64_t n_rows) {
  std::vector<uint8_t> img;
  ParquetColumnDesc d = c;
  if (c.codec == CODEC_ZSTD) {
    check_parquet_column(f, c, n_rows);
    img = zstd_image_host(f, c, n_rows, &d.chunk_len);
    d.chunk = img.data();
  }
  ColumnPlan P = plan_parquet_column(f, d, n_rows);
  int64_t level_vals = 0, index_vals = 0;
  for (auto& r : P.level_runs) level_vals += r.count;
  for (auto& r : P.index_runs) index_vals += r.count;
  uint64_t body_bytes = 0, body_hash = 0xcbf29ce484222325ull;
  for (auto& s : P.bodies) { body_bytes += s.second; body_hash = fnv1a(body_hash, s.first, s.second); }
  char b[640];
  snprintf(b, sizeof b, "{\"pages\":%lld,\"dense\":%lld,\"dict_count\":%lld,\"level_values\":%lld,\"index_values\":%lld,\"level_runs\":%zu,\"index_runs\":%zu,"
                        "\"plain_strings\":%zu,\"dict_pages\":%d,\"plain_pages\":%d,\"body_bytes\":%llu,\"body_fnv1a\":%llu,"
                        "\"delta_pages\":%lld,\"delta_values\":%lld,\"bss_pages\":%lld,\"bss_values\":%lld}",      // at most 547 bytes
           (long long)P.n_pages, (long long)P.dense, (long long)P.dict_count, (long long)level_vals, (long long)index_vals, P.level_runs.size(), P.index_runs.size(),
           P.str_off.size(), P.any_dict_page ? 1 : 0, P.any_plain_page ? 1 : 0, (unsigned long long)body_bytes, (unsigned long long)body_hash,
           (long long)P.delta_pages, (long long)P.delta_values, (long long)P.bss_pages, (long long)P.bss_values);
  return b;
}

}  // namespace sg
