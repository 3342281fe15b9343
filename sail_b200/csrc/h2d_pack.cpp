// h2d_pack.cpp -- the host loops of the packed ingest (h2d.cu), compiled by g++ with function multiversioning: the library is
// built on one machine and runs on another, so every loop exists as an AVX-512, an AVX2 and a baseline clone and glibc's ifunc
// picks at load time.  Plain streaming loops (range scan, narrowing stores) written so that the vectoriser takes them.
#include <cstdint>
#include <cstring>
#if defined(__x86_64__)
#include <immintrin.h>
#endif

#if defined(__x86_64__)
#define SG_MV __attribute__((target_clones("avx512f", "avx2", "default")))
#else
#define SG_MV
#endif

extern "C" {

// Decimal128 piece: min / max of the low words, and whether every high word is the sign extension of its low word
SG_MV void sg_scan_dec128(const int64_t* __restrict p, int64_t n, int64_t* mn_out, int64_t* mx_out, uint64_t* bad_out) {
  int64_t mn = INT64_MAX, mx = INT64_MIN;
  uint64_t bad = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t lo = p[2 * i], hi = p[2 * i + 1];
    bad |= (uint64_t)(hi ^ (lo >> 63));
    mn = lo < mn ? lo : mn;
    mx = lo > mx ? lo : mx;
  }
  *mn_out = mn; *mx_out = mx; *bad_out = bad;
}
SG_MV void sg_scan_i64(const int64_t* __restrict p, int64_t n, int64_t* mn_out, int64_t* mx_out) {
  int64_t mn = INT64_MAX, mx = INT64_MIN;
  for (int64_t i = 0; i < n; ++i) { mn = p[i] < mn ? p[i] : mn; mx = p[i] > mx ? p[i] : mx; }
  *mn_out = mn; *mx_out = mx;
}
SG_MV void sg_scan_i32(const int32_t* __restrict p, int64_t n, int32_t* mn_out, int32_t* mx_out) {
  int32_t mn = INT32_MAX, mx = INT32_MIN;
  for (int64_t i = 0; i < n; ++i) { mn = p[i] < mn ? p[i] : mn; mx = p[i] > mx ? p[i] : mx; }
  *mn_out = mn; *mx_out = mx;
}
SG_MV uint32_t sg_scan_view_maxlen(const uint32_t* __restrict p, int64_t n) {
  uint32_t L = 0;
  for (int64_t i = 0; i < n; ++i) L = p[4 * i] > L ? p[4 * i] : L;
  return L;
}

// deltas against `base`, narrowed to w bytes; `stride` in elements (2 for the low words of Decimal128)
SG_MV void sg_pack_i64(uint8_t* __restrict out, const int64_t* __restrict vals, int64_t stride, int64_t n, int64_t base, int w) {
  const uint64_t b = (uint64_t)base;
  if (stride == 2) {
    switch (w) {
      case 1: for (int64_t i = 0; i < n; ++i) out[i] = (uint8_t)((uint64_t)vals[2 * i] - b); break;
      case 2: { uint16_t* o = reinterpret_cast<uint16_t*>(out); for (int64_t i = 0; i < n; ++i) o[i] = (uint16_t)((uint64_t)vals[2 * i] - b); break; }
      case 4: { uint32_t* o = reinterpret_cast<uint32_t*>(out); for (int64_t i = 0; i < n; ++i) o[i] = (uint32_t)((uint64_t)vals[2 * i] - b); break; }
      default: { uint64_t* o = reinterpret_cast<uint64_t*>(out); for (int64_t i = 0; i < n; ++i) o[i] = (uint64_t)vals[2 * i] - b; }
    }
  } else {
    switch (w) {
      case 1: for (int64_t i = 0; i < n; ++i) out[i] = (uint8_t)((uint64_t)vals[i] - b); break;
      case 2: { uint16_t* o = reinterpret_cast<uint16_t*>(out); for (int64_t i = 0; i < n; ++i) o[i] = (uint16_t)((uint64_t)vals[i] - b); break; }
      case 4: { uint32_t* o = reinterpret_cast<uint32_t*>(out); for (int64_t i = 0; i < n; ++i) o[i] = (uint32_t)((uint64_t)vals[i] - b); break; }
      default: { uint64_t* o = reinterpret_cast<uint64_t*>(out); for (int64_t i = 0; i < n; ++i) o[i] = (uint64_t)vals[i] - b; }
    }
  }
}
SG_MV void sg_pack_i32(uint8_t* __restrict out, const int32_t* __restrict vals, int64_t n, int32_t base, int w) {
  const uint32_t b = (uint32_t)base;
  if (w == 1) for (int64_t i = 0; i < n; ++i) out[i] = (uint8_t)((uint32_t)vals[i] - b);
  else { uint16_t* o = reinterpret_cast<uint16_t*>(out); for (int64_t i = 0; i < n; ++i) o[i] = (uint16_t)((uint32_t)vals[i] - b); }
}
// inline views -> [length byte][L bytes] rows
SG_MV void sg_pack_views(uint8_t* __restrict out, const uint8_t* __restrict views, int64_t n, uint32_t L) {
  if (L == 0) { for (int64_t i = 0; i < n; ++i) out[i] = views[16 * i]; return; }
  if (L == 1) { for (int64_t i = 0; i < n; ++i) { out[2 * i] = views[16 * i]; out[2 * i + 1] = views[16 * i + 4]; } return; }
  const size_t rb = 1 + L;
  for (int64_t i = 0; i < n; ++i) {
    const uint8_t* v = views + 16 * i;
    uint8_t* o = out + rb * (size_t)i;
    o[0] = v[0];
    for (uint32_t k = 0; k < L; ++k) o[1 + k] = v[4 + k];
  }
}


// ---- one-pass variants: pack under an ASSUMED encoding and report what the piece really holds --------------------------------
// The scan + pack pair above reads a piece twice (DRAM, then L2).  A core streams from DRAM at roughly the speed it packs, so the
// ingest is faster when the common case touches every source byte once: the caller guesses (base, width) from a few strided
// samples of the piece, these loops store the narrowed deltas AND reduce min / max / sign-extension on the way, and the caller
// keeps the result if the true range fits the guess (else it re-packs exactly; the piece is in L2 by then).
#define SG_PACKCHK_LOOP(OT, LOAD, EXTRA)                                     \
  { OT* o = reinterpret_cast<OT*>(out);                                      \
    for (int64_t i = 0; i < n; ++i) { const int64_t v = LOAD; EXTRA; mn = v < mn ? v : mn; mx = v > mx ? v : mx; o[i] = (OT)((uint64_t)v - b); } }
SG_MV static void packchk_dec128_generic(uint8_t* __restrict out, const int64_t* __restrict p, int64_t n, int64_t base, int w, int64_t* mn_out, int64_t* mx_out, uint64_t* bad_out) {
  int64_t mn = INT64_MAX, mx = INT64_MIN;
  uint64_t bad = 0;
  const uint64_t b = (uint64_t)base;
  switch (w) {
    case 1: SG_PACKCHK_LOOP(uint8_t, p[2 * i], bad |= (uint64_t)(p[2 * i + 1] ^ (v >> 63))) break;
    case 2: SG_PACKCHK_LOOP(uint16_t, p[2 * i], bad |= (uint64_t)(p[2 * i + 1] ^ (v >> 63))) break;
    default: SG_PACKCHK_LOOP(uint32_t, p[2 * i], bad |= (uint64_t)(p[2 * i + 1] ^ (v >> 63))) break;
  }
  *mn_out = mn; *mx_out = mx; *bad_out = bad;
}
SG_MV void sg_packchk_i64(uint8_t* __restrict out, const int64_t* __restrict p, int64_t n, int64_t base, int w, int64_t* mn_out, int64_t* mx_out) {
  int64_t mn = INT64_MAX, mx = INT64_MIN;
  const uint64_t b = (uint64_t)base;
  switch (w) {
    case 1: SG_PACKCHK_LOOP(uint8_t, p[i], (void)0) break;
    case 2: SG_PACKCHK_LOOP(uint16_t, p[i], (void)0) break;
    default: SG_PACKCHK_LOOP(uint32_t, p[i], (void)0) break;
  }
  *mn_out = mn; *mx_out = mx;
}
SG_MV void sg_packchk_i32(uint8_t* __restrict out, const int32_t* __restrict p, int64_t n, int32_t base, int w, int32_t* mn_out, int32_t* mx_out) {
  int32_t mn = INT32_MAX, mx = INT32_MIN;
  const uint32_t b = (uint32_t)base;
  if (w == 1) { for (int64_t i = 0; i < n; ++i) { const int32_t v = p[i]; mn = v < mn ? v : mn; mx = v > mx ? v : mx; out[i] = (uint8_t)((uint32_t)v - b); } }
  else { uint16_t* o = reinterpret_cast<uint16_t*>(out); for (int64_t i = 0; i < n; ++i) { const int32_t v = p[i]; mn = v < mn ? v : mn; mx = v > mx ? v : mx; o[i] = (uint16_t)((uint32_t)v - b); } }
  *mn_out = mn; *mx_out = mx;
}
// inline views under an assumed maximum length L (0..12); returns the true maximum length of the piece
SG_MV static uint32_t packchk_views_generic(uint8_t* __restrict out, const uint8_t* __restrict views, int64_t n, uint32_t L) {
  uint32_t mxl = 0;
  if (L == 0) { for (int64_t i = 0; i < n; ++i) { const uint32_t l = *reinterpret_cast<const uint32_t*>(views + 16 * i); mxl = l > mxl ? l : mxl; out[i] = (uint8_t)l; } return mxl; }
  if (L == 1) { for (int64_t i = 0; i < n; ++i) { const uint32_t l = *reinterpret_cast<const uint32_t*>(views + 16 * i); mxl = l > mxl ? l : mxl; out[2 * i] = (uint8_t)l; out[2 * i + 1] = views[16 * i + 4]; } return mxl; }
  const size_t rb = 1 + L;
  for (int64_t i = 0; i < n; ++i) {
    const uint8_t* v = views + 16 * i;
    const uint32_t l = *reinterpret_cast<const uint32_t*>(v);
    mxl = l > mxl ? l : mxl;
    uint8_t* o = out + rb * (size_t)i;
    o[0] = (uint8_t)l;
    for (uint32_t k = 0; k < L; ++k) o[1 + k] = v[4 + k];
  }
  return mxl;
}


#if defined(__x86_64__)
// Hand-written AVX-512 forms of the two loops that carry most TPC-H bytes (Decimal128 values; one-character views): the strided
// low/high-word split and the three reductions keep the compiler's vectoriser at ~10 GB/s per core, below what a core streams.
__attribute__((target("avx512f,avx512bw,avx512vl")))
static void packchk_dec128_avx512(uint8_t* __restrict out, const int64_t* __restrict p, int64_t n, int64_t base, int w, int64_t* mn_out, int64_t* mx_out, uint64_t* bad_out) {
  const __m512i idx_lo = _mm512_setr_epi64(0, 2, 4, 6, 8, 10, 12, 14), idx_hi = _mm512_setr_epi64(1, 3, 5, 7, 9, 11, 13, 15);
  const __m512i vb = _mm512_set1_epi64(base);
  __m512i vmn = _mm512_set1_epi64(INT64_MAX), vmx = _mm512_set1_epi64(INT64_MIN), vbad = _mm512_setzero_si512();
  int64_t i = 0;
  for (; i + 16 <= n; i += 16) {
    // a core's line-fill buffers alone limit what one thread streams from DRAM; software prefetches 4 KB ahead add to it
    { const char* pf = reinterpret_cast<const char*>(p + 2 * i) + 4096;
      _mm_prefetch(pf, _MM_HINT_T0); _mm_prefetch(pf + 64, _MM_HINT_T0); _mm_prefetch(pf + 128, _MM_HINT_T0); _mm_prefetch(pf + 192, _MM_HINT_T0); }
    const __m512i a0 = _mm512_loadu_si512(p + 2 * i), a1 = _mm512_loadu_si512(p + 2 * i + 8), a2 = _mm512_loadu_si512(p + 2 * i + 16), a3 = _mm512_loadu_si512(p + 2 * i + 24);
    const __m512i lo0 = _mm512_permutex2var_epi64(a0, idx_lo, a1), hi0 = _mm512_permutex2var_epi64(a0, idx_hi, a1);
    const __m512i lo1 = _mm512_permutex2var_epi64(a2, idx_lo, a3), hi1 = _mm512_permutex2var_epi64(a2, idx_hi, a3);
    vbad = _mm512_or_si512(vbad, _mm512_or_si512(_mm512_xor_si512(hi0, _mm512_srai_epi64(lo0, 63)), _mm512_xor_si512(hi1, _mm512_srai_epi64(lo1, 63))));
    vmn = _mm512_min_epi64(vmn, _mm512_min_epi64(lo0, lo1));
    vmx = _mm512_max_epi64(vmx, _mm512_max_epi64(lo0, lo1));
    const __m512i d0 = _mm512_sub_epi64(lo0, vb), d1 = _mm512_sub_epi64(lo1, vb);
    if (w == 1) {
      _mm_storel_epi64(reinterpret_cast<__m128i*>(out + i), _mm512_cvtepi64_epi8(d0));
      _mm_storel_epi64(reinterpret_cast<__m128i*>(out + i + 8), _mm512_cvtepi64_epi8(d1));
    } else if (w == 2) {
      _mm_storeu_si128(reinterpret_cast<__m128i*>(out + 2 * i), _mm512_cvtepi64_epi16(d0));
      _mm_storeu_si128(reinterpret_cast<__m128i*>(out + 2 * i + 16), _mm512_cvtepi64_epi16(d1));
    } else {
      _mm256_storeu_si256(reinterpret_cast<__m256i*>(out + 4 * i), _mm512_cvtepi64_epi32(d0));
      _mm256_storeu_si256(reinterpret_cast<__m256i*>(out + 4 * i + 32), _mm512_cvtepi64_epi32(d1));
    }
  }
  int64_t mn = _mm512_reduce_min_epi64(vmn), mx = _mm512_reduce_max_epi64(vmx);
  uint64_t bad = (uint64_t)_mm512_reduce_or_epi64(vbad);
  const uint64_t b = (uint64_t)base;
  for (; i < n; ++i) {
    const int64_t v = p[2 * i];
    bad |= (uint64_t)(p[2 * i + 1] ^ (v >> 63));
    mn = v < mn ? v : mn; mx = v > mx ? v : mx;
    const uint64_t d = (uint64_t)v - b;
    if (w == 1) out[i] = (uint8_t)d; else if (w == 2) reinterpret_cast<uint16_t*>(out)[i] = (uint16_t)d; else reinterpret_cast<uint32_t*>(out)[i] = (uint32_t)d;
  }
  *mn_out = mn; *mx_out = mx; *bad_out = bad;
}
// one-character views: [len, c] of 16 views per iteration (4 loads, 4 byte shuffles into disjoint word slots, one 4x4 word transpose)
__attribute__((target("avx512f,avx512bw,avx512vl")))
static uint32_t packchk_views1_avx512(uint8_t* __restrict out, const uint8_t* __restrict views, int64_t n) {
  const char Z = (char)0x80;
  const __m512i sh0 = _mm512_broadcast_i32x4(_mm_setr_epi8(0, 4, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z));
  const __m512i sh1 = _mm512_broadcast_i32x4(_mm_setr_epi8(Z, Z, 0, 4, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z));
  const __m512i sh2 = _mm512_broadcast_i32x4(_mm_setr_epi8(Z, Z, Z, Z, 0, 4, Z, Z, Z, Z, Z, Z, Z, Z, Z, Z));
  const __m512i sh3 = _mm512_broadcast_i32x4(_mm_setr_epi8(Z, Z, Z, Z, Z, Z, 0, 4, Z, Z, Z, Z, Z, Z, Z, Z));
  const __m512i lenmask = _mm512_broadcast_i32x4(_mm_setr_epi32(-1, 0, 0, 0));
  const __m512i qsel = _mm512_setr_epi64(0, 2, 4, 6, 0, 0, 0, 0);
  // after the ORs, 128-bit lane j holds the words of views j, 4+j, 8+j, 12+j: word (4j + k) is view (4k + j)
  const __m256i tr = _mm256_setr_epi16(0, 4, 8, 12, 1, 5, 9, 13, 2, 6, 10, 14, 3, 7, 11, 15);
  __m512i vmx = _mm512_setzero_si512();
  int64_t i = 0;
  for (; i + 16 <= n; i += 16) {
    { const char* pf = reinterpret_cast<const char*>(views + 16 * i) + 4096;
      _mm_prefetch(pf, _MM_HINT_T0); _mm_prefetch(pf + 64, _MM_HINT_T0); _mm_prefetch(pf + 128, _MM_HINT_T0); _mm_prefetch(pf + 192, _MM_HINT_T0); }
    const __m512i v0 = _mm512_loadu_si512(views + 16 * i), v1 = _mm512_loadu_si512(views + 16 * i + 64), v2 = _mm512_loadu_si512(views + 16 * i + 128), v3 = _mm512_loadu_si512(views + 16 * i + 192);
    vmx = _mm512_max_epu32(vmx, _mm512_max_epu32(_mm512_max_epu32(_mm512_and_si512(v0, lenmask), _mm512_and_si512(v1, lenmask)),
                                                 _mm512_max_epu32(_mm512_and_si512(v2, lenmask), _mm512_and_si512(v3, lenmask))));
    // here lane j of v_k is view 4k + j: v_k's bytes go to word slot k of its lane
    const __m512i r = _mm512_or_si512(_mm512_or_si512(_mm512_shuffle_epi8(v0, sh0), _mm512_shuffle_epi8(v1, sh1)),
                                      _mm512_or_si512(_mm512_shuffle_epi8(v2, sh2), _mm512_shuffle_epi8(v3, sh3)));
    const __m256i q = _mm512_castsi512_si256(_mm512_permutexvar_epi64(qsel, r));      // words: lane j, slot k at 4j + k = view 4k + j
    _mm256_storeu_si256(reinterpret_cast<__m256i*>(out + 2 * i), _mm256_permutexvar_epi16(tr, q));
  }
  uint32_t mxl = _mm512_reduce_max_epu32(vmx);
  for (; i < n; ++i) { const uint32_t l = *reinterpret_cast<const uint32_t*>(views + 16 * i); mxl = l > mxl ? l : mxl; out[2 * i] = (uint8_t)l; out[2 * i + 1] = views[16 * i + 4]; }
  return mxl;
}
static bool have_avx512() { static const bool v = __builtin_cpu_supports("avx512f") && __builtin_cpu_supports("avx512bw") && __builtin_cpu_supports("avx512vl"); return v; }
#else
static bool have_avx512() { return false; }
#endif

__attribute__((visibility("default"))) void sg_packchk_dec128(uint8_t* out, const int64_t* p, int64_t n, int64_t base, int w, int64_t* mn_out, int64_t* mx_out, uint64_t* bad_out) {
#if defined(__x86_64__)
  if (have_avx512()) { packchk_dec128_avx512(out, p, n, base, w, mn_out, mx_out, bad_out); return; }
#endif
  packchk_dec128_generic(out, p, n, base, w, mn_out, mx_out, bad_out);
}
__attribute__((visibility("default"))) uint32_t sg_packchk_views(uint8_t* out, const uint8_t* views, int64_t n, uint32_t L) {
#if defined(__x86_64__)
  if (L == 1 && have_avx512()) return packchk_views1_avx512(out, views, n);
#endif
  return packchk_views_generic(out, views, n, L);
}

}  // extern "C"
