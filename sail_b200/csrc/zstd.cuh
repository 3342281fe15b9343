// zstd.cuh -- ZSTD frame decoder (RFC 8878) for the pages of Parquet column chunks (parquet.cu).
//
// One code path serves both sides: the device kernel runs it with a warp as the team (one warp per frame, frames are the unit
// of parallelism because a match may reach back into any earlier block of its frame), sailgpu_parquet_inspect runs it on the
// host with a single thread as the team.  Inside a block the serial parts (Huffman and FSE table builds, the sequence bit
// stream) run on lane 0 and publish their results through the team's ZWork; the four Huffman streams are decoded by four
// lanes at once; every copy (raw / RLE blocks, literal runs, matches) is lane-strided.
//
// Decoded: frames with or without Frame_Content_Size, Single_Segment set or not, an optional content checksum (skipped),
// Raw / RLE / Compressed blocks, literals Raw / RLE / Compressed (1 or 4 streams) / Treeless, sequences in Predefined / RLE /
// FSE_Compressed / Repeat modes, and several frames concatenated in one page body.  Refused: dictionaries and skippable
// frames (ZS_UNSUPPORTED).  Every bit-stream read is checked against its block, every write against the output's length;
// a malformed frame returns ZS_CORRUPT and never reads or writes out of bounds.
#pragma once
#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define ZS_HD __host__ __device__ __forceinline__
#else
#define ZS_HD inline
#endif

namespace sg {
namespace zstd {

enum : int { ZS_OK = 0, ZS_CORRUPT = 1, ZS_UNSUPPORTED = 2 };
constexpr uint32_t kMagic = 0xFD2FB528u;
constexpr uint32_t kBlockMax = 128u << 10;       // Block_Maximum_Size: no block carries more (literals included)
constexpr int kSeqBatch = 64;                     // sequences decoded by lane 0 before the team executes them

ZS_HD int highbit(uint32_t v) {                   // index of the highest set bit (v > 0)
#if defined(__CUDA_ARCH__)
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}
ZS_HD uint32_t le16(const uint8_t* p) { return p[0] | ((uint32_t)p[1] << 8); }
ZS_HD uint32_t le24(const uint8_t* p) { return p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16); }
ZS_HD uint32_t le32(const uint8_t* p) { return le24(p) | ((uint32_t)p[3] << 24); }

// ---- frame header (RFC 8878 3.1.1.1) ---------------------------------------------------------------------------------
struct FrameHeader {
  uint32_t header_len;        // magic included
  uint64_t content_size;      // Frame_Content_Size, when has_content_size
  bool has_content_size, has_checksum;
};
// parses the header of the frame at p[0, n); ZS_UNSUPPORTED for skippable frames and dictionaries
ZS_HD int parse_frame_header(const uint8_t* p, size_t n, FrameHeader* h) {
  if (n < 4) return ZS_CORRUPT;
  const uint32_t magic = le32(p);
  if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) return ZS_UNSUPPORTED;      // skippable frame
  if (magic != kMagic || n < 5) return ZS_CORRUPT;
  const uint32_t fhd = p[4];
  if (fhd & 0x08) return ZS_CORRUPT;                                   // reserved bit
  const bool single = (fhd >> 5) & 1;
  const uint32_t did_size = (fhd & 3) == 3 ? 4 : (fhd & 3);
  const uint32_t fcs_flag = fhd >> 6;
  const uint32_t fcs_size = fcs_flag == 0 ? (single ? 1 : 0) : (1u << fcs_flag);
  size_t q = 5 + (single ? 0 : 1);
  if (q + did_size + fcs_size > n) return ZS_CORRUPT;
  uint32_t did = 0;
  for (uint32_t k = 0; k < did_size; ++k) did |= (uint32_t)p[q + k] << (8 * k);
  if (did != 0) return ZS_UNSUPPORTED;                                 // a dictionary the page does not carry
  q += did_size;
  uint64_t fcs = 0;
  for (uint32_t k = 0; k < fcs_size; ++k) fcs |= (uint64_t)p[q + k] << (8 * k);
  if (fcs_size == 2) fcs += 256;
  h->header_len = (uint32_t)(q + fcs_size);
  h->content_size = fcs;
  h->has_content_size = fcs_size != 0;
  h->has_checksum = (fhd >> 2) & 1;
  return ZS_OK;
}

// ---- bit readers -------------------------------------------------------------------------------------------------------
// Backward stream (RFC 8878 4.1): read from the end towards the start; the last byte's highest set bit is padding.  Bits
// beyond the start read as zeros and drive `left` negative, which every caller checks.
struct BitBwd {
  const uint8_t* p; int64_t n; int64_t left;
  ZS_HD bool init(const uint8_t* s, size_t len) {
    p = s; n = (int64_t)len;
    if (len == 0 || s[len - 1] == 0) return false;
    left = (int64_t)(len - 1) * 8 + highbit(s[len - 1]);
    return true;
  }
  ZS_HD uint64_t load5(int64_t byte) const {
    uint64_t w = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) if (byte + k < n) w |= (uint64_t)p[byte + k] << (8 * k);
    return w;
  }
  ZS_HD uint32_t peek(int nb) const {            // nb <= 32
    if (nb == 0 || left <= 0) return 0;
    const int64_t lo = left - nb;
    if (lo >= 0) return (uint32_t)((load5(lo >> 3) >> (lo & 7)) & ((1ull << nb) - 1));
    return (uint32_t)((load5(0) & ((1ull << left) - 1)) << (-lo));
  }
  ZS_HD uint32_t read(int nb) { const uint32_t v = peek(nb); left -= nb; return v; }
};

// Forward little-endian stream (FSE table descriptions), bounded by n bytes
struct BitFwd {
  const uint8_t* p; size_t n; size_t bit;
  ZS_HD uint32_t peek(int nb) const {            // nb <= 24
    const size_t b = bit >> 3;
    uint32_t w = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) if (b + k < n) w |= (uint32_t)p[b + k] << (8 * k);
    return (w >> (bit & 7)) & ((1u << nb) - 1);
  }
};

// ---- FSE (RFC 8878 4.1.1) ------------------------------------------------------------------------------------------------
struct FseEntry { uint16_t base; uint8_t sym; uint8_t nb; };

// reads an FSE table description of at most `max_sym` + 1 symbols and accuracy <= max_log; returns the bytes used, or 0
ZS_HD size_t read_fse_counts(const uint8_t* src, size_t n, int max_sym, int max_log, int16_t* norm, int* n_sym, int* log) {
  if (n == 0) return 0;
  BitFwd b{src, n, 0};
  const int acc = (int)b.peek(4) + 5; b.bit += 4;
  if (acc > max_log) return 0;
  int remaining = (1 << acc) + 1, threshold = 1 << acc, nbits = acc + 1, sym = 0;
  bool prev0 = false;
  while (remaining > 1 && sym <= max_sym) {
    if (prev0) {                                 // repeat flags: 2 bits each, 3 = "three more zeros and another flag"
      int zeros = 0;
      for (;;) {
        const uint32_t r = b.peek(2); b.bit += 2;
        zeros += (int)r;
        if (r != 3) break;
        if ((b.bit >> 3) > n) return 0;
      }
      if (sym + zeros > max_sym + 1) return 0;
      for (int k = 0; k < zeros; ++k) norm[sym++] = 0;
      if (sym > max_sym) break;
    }
    const int maxv = 2 * threshold - 1 - remaining;
    int count;
    const uint32_t low = b.peek(nbits - 1);
    if ((int)low < maxv) { count = (int)low; b.bit += nbits - 1; }
    else { count = (int)b.peek(nbits); if (count >= threshold) count -= maxv; b.bit += nbits; }
    --count;                                     // -1: "less than 1" probability
    remaining -= count < 0 ? -count : count;
    norm[sym++] = (int16_t)count;
    prev0 = count == 0;
    while (remaining < threshold && threshold > 1) { --nbits; threshold >>= 1; }
    if (((b.bit + 7) >> 3) > n) return 0;
  }
  if (remaining != 1 || ((b.bit + 7) >> 3) > n) return 0;
  *n_sym = sym; *log = acc;
  return (b.bit + 7) >> 3;
}

// decoding table from normalized counts; `next` is scratch for n_sym entries; false on an inconsistent distribution
ZS_HD bool build_fse(const int16_t* norm, int n_sym, int log, FseEntry* t, uint16_t* next) {
  const uint32_t size = 1u << log;
  int high = (int)size - 1;
  for (int s = 0; s < n_sym; ++s) {
    if (norm[s] == -1) { if (high < 0) return false; t[high--].sym = (uint8_t)s; next[s] = 1; }
    else next[s] = (uint16_t)norm[s];
  }
  const uint32_t step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  uint32_t pos = 0;
  for (int s = 0; s < n_sym; ++s) {
    for (int i = 0; i < norm[s]; ++i) {
      t[pos].sym = (uint8_t)s;
      do pos = (pos + step) & mask; while ((int)pos > high);
    }
  }
  if (pos != 0) return false;
  for (uint32_t u = 0; u < size; ++u) {
    const uint32_t ns = next[t[u].sym]++;
    if (ns == 0) return false;
    const int nb = log - highbit(ns);
    t[u].nb = (uint8_t)nb;
    t[u].base = (uint16_t)((ns << nb) - size);
  }
  return true;
}

// ---- sequence codes (RFC 8878 3.1.1.3.2.1) ---------------------------------------------------------------------------------
// codes 16..35 of Literals_Length and 32..52 of Match_Length: baseline and extra bits (below them the code is the value,
// plus 3 for match lengths)
#define ZS_LL_BASE {16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536}
#define ZS_LL_BITS {1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16}
#define ZS_ML_BASE {35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539}
#define ZS_ML_BITS {1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16}
#if defined(__CUDACC__)
static __constant__ uint32_t kLLBaseD[20] = ZS_LL_BASE, kMLBaseD[21] = ZS_ML_BASE;
static __constant__ uint8_t kLLBitsD[20] = ZS_LL_BITS, kMLBitsD[21] = ZS_ML_BITS;
#endif
static const uint32_t kLLBaseH[20] = ZS_LL_BASE, kMLBaseH[21] = ZS_ML_BASE;
static const uint8_t kLLBitsH[20] = ZS_LL_BITS, kMLBitsH[21] = ZS_ML_BITS;
ZS_HD void ll_code(int c, uint32_t* base, int* bits) {
  if (c < 16) { *base = (uint32_t)c; *bits = 0; return; }
#if defined(__CUDA_ARCH__)
  *base = kLLBaseD[c - 16]; *bits = kLLBitsD[c - 16];
#else
  *base = kLLBaseH[c - 16]; *bits = kLLBitsH[c - 16];
#endif
}
ZS_HD void ml_code(int c, uint32_t* base, int* bits) {
  if (c < 32) { *base = (uint32_t)c + 3; *bits = 0; return; }
#if defined(__CUDA_ARCH__)
  *base = kMLBaseD[c - 32]; *bits = kMLBitsD[c - 32];
#else
  *base = kMLBaseH[c - 32]; *bits = kMLBitsH[c - 32];
#endif
}
enum { LL_MAX = 35, ML_MAX = 52, OF_MAX = 31, LL_LOG = 9, ML_LOG = 9, OF_LOG = 8 };
// predefined distributions (RFC 8878 3.1.1.3.2.2)
ZS_HD void predefined(int kind, int16_t* norm, int* n_sym, int* log) {
  const int8_t LL[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
  const int8_t ML[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                         1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
  const int8_t OF[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
  const int8_t* src = kind == 0 ? LL : kind == 1 ? OF : ML;
  *n_sym = kind == 0 ? 36 : kind == 1 ? 29 : 53;
  *log = kind == 1 ? 5 : 6;
  for (int s = 0; s < *n_sym; ++s) norm[s] = src[s];
}

// ---- per-team decoder state --------------------------------------------------------------------------------------------
struct HufEntry { uint8_t sym, nb; };
struct ZWork {
  FseEntry ll[1 << LL_LOG], of[1 << OF_LOG], ml[1 << ML_LOG];
  HufEntry huf[1 << 11];
  union {
    struct { int16_t norm[ML_MAX + 1]; uint16_t next[ML_MAX + 1]; } fse;
    struct { FseEntry t[64]; int16_t norm[16]; uint16_t next[16]; uint8_t w[256]; uint32_t rank[13]; } huf;
  } tmp;
  uint32_t seq_ll[kSeqBatch], seq_ml[kSeqBatch], seq_of[kSeqBatch];
  uint32_t rep[3];
  int ll_log, of_log, ml_log, huf_bits;       // -1: no table yet (Repeat / Treeless are corrupt then)
  int status, n_batch;                        // lane 0 -> team
  uint32_t hdr_len;                           // bytes of the Huffman tree description
  int stream_status[4];
};

// Huffman tree description (RFC 8878 4.2.1) -> w->huf / w->huf_bits; returns bytes used or 0
ZS_HD size_t build_huffman(ZWork* w, const uint8_t* src, size_t n) {
  if (n == 0) return 0;
  uint8_t* wt = w->tmp.huf.w;
  const uint32_t hb = src[0];
  int nw = 0;
  size_t used;
  if (hb >= 128) {                              // direct: 4-bit weights
    nw = (int)hb - 127;
    used = 1 + (size_t)(nw + 1) / 2;
    if (used > n) return 0;
    for (int i = 0; i < nw; ++i) wt[i] = (uint8_t)((i & 1) ? (src[1 + i / 2] & 15) : (src[1 + i / 2] >> 4));
  } else {                                      // FSE-compressed weights, two interleaved states
    used = 1 + hb;
    if (used > n || hb == 0) return 0;
    int ns, log;
    const size_t h = read_fse_counts(src + 1, hb, 15, 6, w->tmp.huf.norm, &ns, &log);
    if (!h || !build_fse(w->tmp.huf.norm, ns, log, w->tmp.huf.t, w->tmp.huf.next)) return 0;
    BitBwd b;
    if (!b.init(src + 1 + h, hb - h)) return 0;
    const FseEntry* t = w->tmp.huf.t;
    uint32_t s1 = b.read(log), s2 = b.read(log);
    if (b.left < 0) return 0;
    for (;;) {
      if (nw > 253) return 0;
      wt[nw++] = t[s1].sym; s1 = t[s1].base + b.read(t[s1].nb);
      if (b.left < 0) { wt[nw++] = t[s2].sym; break; }
      wt[nw++] = t[s2].sym; s2 = t[s2].base + b.read(t[s2].nb);
      if (b.left < 0) { wt[nw++] = t[s1].sym; break; }
    }
  }
  // the last symbol's weight is implied: it completes the sum of 2^(w-1) to a power of two
  uint32_t sum = 0;
  for (int i = 0; i < nw; ++i) { if (wt[i] > 11) return 0; if (wt[i]) sum += 1u << (wt[i] - 1); }
  if (sum == 0 || nw > 255) return 0;
  const int max_bits = highbit(sum) + 1;
  const uint32_t left = (1u << max_bits) - sum;
  if (max_bits > 11 || (left & (left - 1))) return 0;
  wt[nw++] = (uint8_t)(highbit(left) + 1);
  // canonical codes: fill by ascending weight, ascending symbol; a symbol of weight k owns 2^(k-1) consecutive entries
  uint32_t* rank = w->tmp.huf.rank;
  for (int k = 0; k <= 12; ++k) rank[k] = 0;
  for (int i = 0; i < nw; ++i) rank[wt[i]]++;
  uint32_t pos = 0;
  for (int k = 1; k <= max_bits; ++k) { const uint32_t c = rank[k]; rank[k] = pos; pos += c << (k - 1); }
  if (pos != (1u << max_bits)) return 0;
  for (int i = 0; i < nw; ++i) {
    const int k = wt[i];
    if (!k) continue;
    const uint32_t cnt = 1u << (k - 1);
    const HufEntry e{(uint8_t)i, (uint8_t)(max_bits + 1 - k)};
    for (uint32_t j = 0; j < cnt; ++j) w->huf[rank[k] + j] = e;
    rank[k] += cnt;
  }
  w->huf_bits = max_bits;
  return used;
}

// one Huffman stream -> out[0, len); ZS_OK only when the stream is consumed exactly
ZS_HD int decode_huf_stream(const ZWork* w, const uint8_t* src, size_t n, uint8_t* out, uint32_t len) {
  BitBwd b;
  if (!b.init(src, n)) return ZS_CORRUPT;
  const int mb = w->huf_bits;
  for (uint32_t i = 0; i < len; ++i) {
    const HufEntry e = w->huf[b.peek(mb)];
    out[i] = e.sym;
    b.left -= e.nb;
    if (b.left < 0) return ZS_CORRUPT;
  }
  return b.left == 0 ? ZS_OK : ZS_CORRUPT;
}

// one table of the sequences section (mode 0..3) -> t; returns bytes used or -1
ZS_HD int64_t sequence_table(ZWork* w, int kind, int mode, const uint8_t* src, size_t n, FseEntry* t, int* log) {
  const int max_sym = kind == 0 ? LL_MAX : kind == 1 ? OF_MAX : ML_MAX, max_log = kind == 0 ? LL_LOG : kind == 1 ? OF_LOG : ML_LOG;
  int ns, lg;
  if (mode == 0) {
    predefined(kind, w->tmp.fse.norm, &ns, &lg);
    if (!build_fse(w->tmp.fse.norm, ns, lg, t, w->tmp.fse.next)) return -1;
    *log = lg;
    return 0;
  }
  if (mode == 1) {
    if (n < 1 || src[0] > max_sym) return -1;
    t[0] = FseEntry{0, src[0], 0};
    *log = 0;
    return 1;
  }
  if (mode == 3) return *log >= 0 ? 0 : -1;
  const size_t h = read_fse_counts(src, n, max_sym, max_log, w->tmp.fse.norm, &ns, &lg);
  if (!h || !build_fse(w->tmp.fse.norm, ns, lg, t, w->tmp.fse.next)) return -1;
  *log = lg;
  return (int64_t)h;
}

// ---- teams ---------------------------------------------------------------------------------------------------------------
struct SerialTeam {                               // the host: one thread
  static constexpr int size = 1;
  int lane = 0;
  ZS_HD void sync() const {}
};
struct WarpTeam {                                 // the device: one warp, all 32 lanes call every team function
  static constexpr int size = 32;
  int lane;
  ZS_HD void sync() const {
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
  }
};

// match copy: out[op + i] = out[op - off + i]; with off < ml the source overlaps the bytes being written and repeats with
// period off, so out[op + i] = out[op - off + i % off] lets every lane copy independently
template <class T>
ZS_HD void copy_match(const T& t, uint8_t* out, size_t op, uint32_t off, uint32_t ml) {
  const uint8_t* src = out + op - off;
  if (off >= ml) { for (uint32_t i = t.lane; i < ml; i += T::size) out[op + i] = src[i]; }
  else { for (uint32_t i = t.lane; i < ml; i += T::size) out[op + i] = src[i % off]; }
}
template <class T>
ZS_HD void copy_bytes(const T& t, uint8_t* dst, const uint8_t* src, uint32_t n) {
  for (uint32_t i = t.lane; i < n; i += T::size) dst[i] = src[i];
}

// One Compressed block: src[0, n) -> out[op, ...), bounded by cap.  frame_start: first byte of the frame's output (matches
// may not reach before it).  lits: kBlockMax bytes of scratch.  Sets *produced.  Every lane returns the same status.
template <class T>
ZS_HD int decode_block(const T& t, ZWork* w, const uint8_t* src, size_t n, uint8_t* out, size_t op, size_t cap, size_t frame_start, uint8_t* lits,
                       size_t* produced) {
  // ---- literals section
  if (n < 1) return ZS_CORRUPT;
  const int lt = src[0] & 3, sf = (src[0] >> 2) & 3;
  uint32_t regen = 0, csize = 0, hlen = 0;
  int n_streams = 1;
  if (lt < 2) {
    if (sf == 0 || sf == 2) { regen = src[0] >> 3; hlen = 1; }
    else if (sf == 1) { if (n < 2) return ZS_CORRUPT; regen = (src[0] >> 4) + ((uint32_t)src[1] << 4); hlen = 2; }
    else { if (n < 3) return ZS_CORRUPT; regen = (src[0] >> 4) + ((uint32_t)src[1] << 4) + ((uint32_t)src[2] << 12); hlen = 3; }
    csize = lt == 0 ? regen : 1;
  } else {
    if (sf < 2) { if (n < 3) return ZS_CORRUPT; const uint32_t h = le24(src); regen = (h >> 4) & 0x3FF; csize = (h >> 14) & 0x3FF; hlen = 3; n_streams = sf == 0 ? 1 : 4; }
    else if (sf == 2) { if (n < 4) return ZS_CORRUPT; const uint32_t h = le32(src); regen = (h >> 4) & 0x3FFF; csize = (h >> 18) & 0x3FFF; hlen = 4; n_streams = 4; }
    else { if (n < 5) return ZS_CORRUPT; const uint64_t h = le32(src) | ((uint64_t)src[4] << 32); regen = (uint32_t)(h >> 4) & 0x3FFFF; csize = (uint32_t)(h >> 22) & 0x3FFFF; hlen = 5; n_streams = 4; }
  }
  if (regen > kBlockMax || (size_t)hlen + csize > n) return ZS_CORRUPT;
  const uint8_t* lit = lits;
  if (lt == 0) lit = src + hlen;
  else if (lt == 1) { for (uint32_t i = t.lane; i < regen; i += T::size) lits[i] = src[hlen]; }
  else {
    const uint8_t* ls = src + hlen;
    if (t.lane == 0) {
      w->status = ZS_OK; w->hdr_len = 0;
      if (lt == 2) {
        const size_t used = build_huffman(w, ls, csize);
        if (!used) w->status = ZS_CORRUPT; else w->hdr_len = (uint32_t)used;
      } else if (w->huf_bits < 0) w->status = ZS_CORRUPT;          // Treeless without an earlier tree
    }
    t.sync();
    if (w->status) return w->status;
    const uint8_t* ss = ls + w->hdr_len;
    const uint32_t sn = csize - w->hdr_len;
    if (n_streams == 1) {
      if (t.lane == 0) w->stream_status[0] = decode_huf_stream(w, ss, sn, lits, regen);
      t.sync();
      if (w->stream_status[0]) return ZS_CORRUPT;
    } else {
      if (sn < 6) return ZS_CORRUPT;
      const uint32_t s1 = le16(ss), s2 = le16(ss + 2), s3 = le16(ss + 4);
      const uint32_t seg = (regen + 3) / 4;
      if ((uint64_t)s1 + s2 + s3 + 6 > sn || 3ull * seg > regen) return ZS_CORRUPT;
      const uint32_t s4 = sn - 6 - s1 - s2 - s3;
      const uint32_t sz[4] = {s1, s2, s3, s4};
      for (int s = t.lane; s < 4; s += T::size) {
        const uint8_t* p = ss + 6;
        for (int k = 0; k < s; ++k) p += sz[k];
        w->stream_status[s] = decode_huf_stream(w, p, sz[s], lits + (size_t)s * seg, s < 3 ? seg : regen - 3 * seg);
      }
      t.sync();
      if (w->stream_status[0] | w->stream_status[1] | w->stream_status[2] | w->stream_status[3]) return ZS_CORRUPT;
    }
  }
  t.sync();
  src += hlen + csize; n -= hlen + csize;

  // ---- sequences section header
  if (n < 1) return ZS_CORRUPT;
  uint32_t nseq = src[0], sh = 1;
  if (nseq >= 128) {
    if (nseq < 255) { if (n < 2) return ZS_CORRUPT; nseq = ((nseq - 128) << 8) + src[1]; sh = 2; }
    else { if (n < 3) return ZS_CORRUPT; nseq = src[1] + ((uint32_t)src[2] << 8) + 0x7F00; sh = 3; }
  }
  size_t lp = 0;                                  // literals consumed
  size_t o = op;
  if (nseq > 0) {
    if (n < sh + 1) return ZS_CORRUPT;
    const uint32_t modes = src[sh];
    if (modes & 3) return ZS_CORRUPT;
    const uint8_t* q = src + sh + 1;
    const uint8_t* qend = src + n;
    // lane 0 builds the tables and then decodes sequences in batches; the team executes each batch
    BitBwd b;
    uint32_t sll = 0, sof = 0, sml = 0, done = 0;
    if (t.lane == 0) {
      w->status = ZS_OK;
      const int mode_of[3] = {(int)(modes >> 6), (int)((modes >> 4) & 3), (int)((modes >> 2) & 3)};
      FseEntry* tabs[3] = {w->ll, w->of, w->ml};
      int* logs[3] = {&w->ll_log, &w->of_log, &w->ml_log};
      for (int k = 0; k < 3 && !w->status; ++k) {
        const int64_t used = sequence_table(w, k, mode_of[k], q, (size_t)(qend - q), tabs[k], logs[k]);
        if (used < 0) w->status = ZS_CORRUPT; else q += used;
      }
      if (!w->status && !b.init(q, (size_t)(qend - q))) w->status = ZS_CORRUPT;
      if (!w->status) {
        sll = b.read(w->ll_log); sof = b.read(w->of_log); sml = b.read(w->ml_log);
        if (b.left < 0) w->status = ZS_CORRUPT;
      }
    }
    t.sync();
    if (w->status) return w->status;
    while (done < nseq) {
      if (t.lane == 0) {
        const int cnt = (int)((nseq - done) < (uint32_t)kSeqBatch ? (nseq - done) : (uint32_t)kSeqBatch);
        for (int i = 0; i < cnt && !w->status; ++i) {
          const int ofc = w->of[sof].sym, mlc = w->ml[sml].sym, llc = w->ll[sll].sym;
          if (ofc > OF_MAX) { w->status = ZS_CORRUPT; break; }
          uint32_t llb, mlb; int lln, mln;
          ll_code(llc, &llb, &lln); ml_code(mlc, &mlb, &mln);
          const uint32_t ofv = (1u << ofc) + b.read(ofc);
          const uint32_t ml = mlb + b.read(mln);
          const uint32_t ll = llb + b.read(lln);
          uint32_t off;
          if (ofv > 3) { off = ofv - 3; w->rep[2] = w->rep[1]; w->rep[1] = w->rep[0]; w->rep[0] = off; }
          else {
            const uint32_t idx = ofv - 1 + (ll == 0 ? 1 : 0);
            if (idx == 0) off = w->rep[0];
            else {
              off = idx == 3 ? w->rep[0] - 1 : w->rep[idx];
              if (idx > 1) w->rep[2] = w->rep[1];
              w->rep[1] = w->rep[0]; w->rep[0] = off;
            }
          }
          w->seq_ll[i] = ll; w->seq_ml[i] = ml; w->seq_of[i] = off;
          if (done + i + 1 < nseq) {               // state updates: LL, ML, OF
            sll = w->ll[sll].base + b.read(w->ll[sll].nb);
            sml = w->ml[sml].base + b.read(w->ml[sml].nb);
            sof = w->of[sof].base + b.read(w->of[sof].nb);
          }
          if (b.left < 0) w->status = ZS_CORRUPT;
        }
        if (!w->status && done + cnt == nseq && b.left != 0) w->status = ZS_CORRUPT;
        w->n_batch = cnt;
      }
      t.sync();
      if (w->status) return w->status;
      const int cnt = w->n_batch;
      for (int i = 0; i < cnt; ++i) {
        const uint32_t ll = w->seq_ll[i], ml = w->seq_ml[i], off = w->seq_of[i];
        if (lp + ll > regen || o + ll + ml > cap || (o + ll - op) + ml > kBlockMax) return ZS_CORRUPT;
        copy_bytes(t, out + o, lit + lp, ll);
        o += ll; lp += ll;
        if (off == 0 || off > o - frame_start) return ZS_CORRUPT;
        t.sync();
        copy_match(t, out, o, off, ml);
        o += ml;
        t.sync();
      }
      done += (uint32_t)cnt;
    }
  }
  // the literals after the last sequence
  const uint32_t rest = (uint32_t)(regen - lp);
  if (o + rest > cap || (o + rest - op) > kBlockMax) return ZS_CORRUPT;
  copy_bytes(t, out + o, lit + lp, rest);
  o += rest;
  t.sync();
  *produced = o - op;
  return ZS_OK;
}

// Every frame of src[0, n) -> out[0, cap): ZS_OK only when the frames produce exactly cap bytes.  All lanes of the team call
// it with the same arguments and return the same status.
template <class T>
ZS_HD int decode_frames(const T& t, ZWork* w, const uint8_t* src, size_t n, uint8_t* out, size_t cap, uint8_t* lits) {
  size_t ip = 0, op = 0;
  while (ip < n) {
    FrameHeader fh;
    const int hs = parse_frame_header(src + ip, n - ip, &fh);
    if (hs) return hs;
    ip += fh.header_len;
    const size_t frame_start = op;
    if (t.lane == 0) { w->rep[0] = 1; w->rep[1] = 4; w->rep[2] = 8; w->ll_log = w->of_log = w->ml_log = w->huf_bits = -1; }
    t.sync();
    for (;;) {
      if (ip + 3 > n) return ZS_CORRUPT;
      const uint32_t bh = le24(src + ip);
      ip += 3;
      const bool last = bh & 1;
      const uint32_t type = (bh >> 1) & 3, size = bh >> 3;
      if (type == 0) {                            // Raw
        if (size > kBlockMax || ip + size > n || op + size > cap) return ZS_CORRUPT;
        copy_bytes(t, out + op, src + ip, size);
        ip += size; op += size;
      } else if (type == 1) {                     // RLE: one byte, repeated `size` times
        if (size > kBlockMax || ip + 1 > n || op + size > cap) return ZS_CORRUPT;
        const uint8_t v = src[ip];
        for (uint32_t i = t.lane; i < size; i += T::size) out[op + i] = v;
        ip += 1; op += size;
      } else if (type == 2) {
        if (size > kBlockMax || ip + size > n) return ZS_CORRUPT;
        size_t produced = 0;
        const int st = decode_block(t, w, src + ip, size, out, op, cap, frame_start, lits, &produced);
        if (st) return st;
        ip += size; op += produced;
      } else return ZS_CORRUPT;
      t.sync();
      if (last) break;
    }
    if (fh.has_checksum) { if (ip + 4 > n) return ZS_CORRUPT; ip += 4; }
    if (fh.has_content_size && op - frame_start != fh.content_size) return ZS_CORRUPT;
  }
  return op == cap ? ZS_OK : ZS_CORRUPT;
}

}  // namespace zstd
}  // namespace sg
