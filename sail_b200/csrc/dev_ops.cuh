// dev_ops.cuh -- small device helpers shared by the interpreter kernel (pipeline.cu) and the runtime of the
// specialised (NVRTC-compiled) pipeline kernels (jit_rt.cuh): wrapping arithmetic, date/LIKE helpers, accumulator
// identities and combiners, 128-bit atomics, the ordered compaction of a tile.
#pragma once
#include "dev_util.cuh"
#include "vm.h"

namespace sg {

struct OpAdd { template <typename T> static __device__ __forceinline__ T f(T a, T b) { return a + b; } };
struct OpSub { template <typename T> static __device__ __forceinline__ T f(T a, T b) { return a - b; } };
struct OpMul { template <typename T> static __device__ __forceinline__ T f(T a, T b) { return a * b; } };
template <> __device__ __forceinline__ int32_t OpAdd::f<int32_t>(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
template <> __device__ __forceinline__ int32_t OpSub::f<int32_t>(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }
template <> __device__ __forceinline__ int32_t OpMul::f<int32_t>(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }
template <> __device__ __forceinline__ int64_t OpAdd::f<int64_t>(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
template <> __device__ __forceinline__ int64_t OpSub::f<int64_t>(int64_t a, int64_t b) { return (int64_t)((uint64_t)a - (uint64_t)b); }
template <> __device__ __forceinline__ int64_t OpMul::f<int64_t>(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }
template <> __device__ __forceinline__ i128 OpAdd::f<i128>(i128 a, i128 b) { return (i128)((u128)a + (u128)b); }
template <> __device__ __forceinline__ i128 OpSub::f<i128>(i128 a, i128 b) { return (i128)((u128)a - (u128)b); }
template <> __device__ __forceinline__ i128 OpMul::f<i128>(i128 a, i128 b) { return (i128)((u128)a * (u128)b); }

struct CmpEq { template <typename T> static __device__ __forceinline__ bool f(T a, T b) { return a == b; } };
struct CmpNe { template <typename T> static __device__ __forceinline__ bool f(T a, T b) { return a != b; } };
struct CmpLt { template <typename T> static __device__ __forceinline__ bool f(T a, T b) { return a < b; } };
struct CmpLe { template <typename T> static __device__ __forceinline__ bool f(T a, T b) { return a <= b; } };
struct CmpGt { template <typename T> static __device__ __forceinline__ bool f(T a, T b) { return a > b; } };
struct CmpGe { template <typename T> static __device__ __forceinline__ bool f(T a, T b) { return a >= b; } };

// days since 1970-01-01 -> civil (year, month, day)
__device__ __forceinline__ void civil_from_days(int32_t z0, int& y, int& m, int& d) {
  int64_t z = (int64_t)z0 + 719468;
  int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  int64_t doe = z - era * 146097;
  int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  int64_t yy = yoe + era * 400;
  int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  int64_t mp = (5 * doy + 2) / 153;
  d = (int)(doy - (153 * mp + 2) / 5 + 1);
  m = (int)(mp < 10 ? mp + 3 : mp - 9);
  y = (int)(m <= 2 ? yy + 1 : yy);
}
// civil (year, month, day) -> days since 1970-01-01: the inverse of civil_from_days
__device__ __forceinline__ int32_t days_from_civil(int y, int m, int d) {
  y -= m <= 2;
  const int era = (y >= 0 ? y : y - 399) / 400;
  const int yoe = y - era * 400;
  const int doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;
  const int doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + doe - 719468;
}

// ---- timestamps (Int64 counts of UPS units per second since the epoch) --------------------------------------------------
// OP_TS_PART / OP_TS_TRUNC read wall-clock time in a fixed-offset zone: `off` is the offset from UTC in units.  The unit is a
// template argument, so every division below is by a compile-time constant and becomes a multiply-high: the interpreter
// dispatches once per instruction on the unit (pipeline.cu: vm_ts), the specialised kernel names it in the generated code.
// The calendar parts go through 32-bit day counts: exact within Date32's range (about 5.8 million years around the epoch).
template <int64_t D> __device__ __forceinline__ int64_t floor_div_c(int64_t a) {
  const int64_t q = a / D;
  return a - q * D < 0 ? q - 1 : q;
}
template <int64_t UPS> __device__ __forceinline__ int64_t ts_part_u(int64_t v, int part, int64_t off) {
  constexpr int64_t DAY = 86400 * UPS;
  const int64_t local = (int64_t)((uint64_t)v + (uint64_t)off);
  const int64_t days = floor_div_c<DAY>(local);
  const int64_t tod = local - days * DAY;      // [0, DAY)
  switch (part) {
    case TS_HOUR: return tod / (3600 * UPS);
    case TS_MINUTE: return (tod / (60 * UPS)) % 60;
    case TS_SECOND: {                           // microsecond within the minute (the unscaled Decimal128(8,6) of Spark's second)
      const int64_t r = tod % (60 * UPS);
      if constexpr (UPS <= 1000000) return r * (1000000 / UPS);
      else return r / (UPS / 1000000);
    }
    case TS_DAYS: return days;
    default: break;
  }
  int y, m, d;
  civil_from_days((int32_t)days, y, m, d);
  return part == TS_YEAR ? y : part == TS_QUARTER ? (m - 1) / 3 + 1 : part == TS_MONTH ? m : d;
}
template <int64_t UPS> __device__ __forceinline__ int64_t ts_trunc_u(int64_t v, int part, int64_t off) {
  constexpr int64_t DAY = 86400 * UPS;
  const int64_t local = (int64_t)((uint64_t)v + (uint64_t)off);
  const int64_t days = floor_div_c<DAY>(local);
  const int64_t tod = local - days * DAY;
  int64_t t;
  switch (part) {
    case TS_SECOND: t = local - tod % UPS; break;
    case TS_MINUTE: t = local - tod % (60 * UPS); break;
    case TS_HOUR: t = local - tod % (3600 * UPS); break;
    case TS_DAY: t = days * DAY; break;
    case TS_WEEK: t = (days - (days + 3 - floor_div_c<7>(days + 3) * 7)) * DAY; break;    // ISO weeks start on Monday; 1970-01-01 was a Thursday
    default: {
      int y, m, d;
      civil_from_days((int32_t)days, y, m, d);
      m = part == TS_YEAR ? 1 : part == TS_QUARTER ? (m - 1) / 3 * 3 + 1 : m;
      t = (int64_t)days_from_civil(y, m, 1) * DAY;
    }
  }
  return (int64_t)((uint64_t)t - (uint64_t)off);
}

__device__ __forceinline__ bool like_match(const uint8_t* s, uint32_t n, const uint8_t* p, uint32_t m, int cls) {
  switch (cls) {
    case LIKE_EXACT:
      if (n != m) return false;
      for (uint32_t i = 0; i < m; ++i) if (s[i] != p[i]) return false;
      return true;
    case LIKE_PREFIX:
      if (n < m) return false;
      for (uint32_t i = 0; i < m; ++i) if (s[i] != p[i]) return false;
      return true;
    case LIKE_SUFFIX:
      if (n < m) return false;
      for (uint32_t i = 0; i < m; ++i) if (s[n - m + i] != p[i]) return false;
      return true;
    case LIKE_CONTAINS:
      if (n < m) return false;
      for (uint32_t st = 0; st + m <= n; ++st) {
        uint32_t i = 0;
        while (i < m && s[st + i] == p[i]) ++i;
        if (i == m) return true;
      }
      return false;
    default: {
      // generic %/_ matcher with single backtrack point (pattern bytes: '%' any run, '_' one byte, '\\' escape)
      uint32_t si = 0, pi = 0, star_p = 0xFFFFFFFFu, star_s = 0;
      while (si < n) {
        if (pi < m && p[pi] == '\\' && pi + 1 < m && p[pi + 1] == s[si]) { pi += 2; ++si; }
        else if (pi < m && p[pi] != '%' && p[pi] != '\\' && (p[pi] == '_' || p[pi] == s[si])) { ++pi; ++si; }
        else if (pi < m && p[pi] == '%') { star_p = pi++; star_s = si; }
        else if (star_p != 0xFFFFFFFFu) { pi = star_p + 1; si = ++star_s; }
        else return false;
      }
      while (pi < m && p[pi] == '%') ++pi;
      return pi == m;
    }
  }
}

__device__ __forceinline__ uint64_t load_key_word(const uint8_t* p, int width) {
  switch (width) {
    case 1: return *p;
    case 4: return (uint64_t)(uint32_t)lds<int32_t>(p);   // zero-extended: equality domain only
    default: return lds<uint64_t>(p);
  }
}

struct KeyRegs { uint64_t w[MAX_KEY_WORDS]; };

enum : uint32_t { ST_EMPTY = 0, ST_LOCKED = 1, ST_READY = 2 };

struct AccVal { i128 i; double f; bool valid; };

__device__ __forceinline__ void atomic_add_i128(uint64_t* w, i128 v) {
  unsigned long long lo = (unsigned long long)(u128)v, hi = (unsigned long long)((u128)v >> 64);
  unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long*>(w), lo);
  unsigned long long carry = (old + lo) < old ? 1ull : 0ull;
  if (hi + carry) atomicAdd(reinterpret_cast<unsigned long long*>(w + 1), hi + carry);
}
__device__ __forceinline__ void atomic_minmax_i128(uint64_t* w, i128 v, bool is_min) {
  u128 cur = ((u128)w[1] << 64) | w[0];
  for (;;) {
    i128 c = (i128)cur;
    if (is_min ? (c <= v) : (c >= v)) return;
    u128 prev = atomic_cas_128(w, cur, (u128)v);
    if (prev == cur) return;
    cur = prev;
  }
}
__device__ __forceinline__ void atomic_minmax_f64(uint64_t* w, double v, bool is_min) {
  unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(w);
  for (;;) {
    double c = __longlong_as_double((long long)cur);
    if (is_min ? (c <= v) : (c >= v)) return;
    unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(w), cur, (unsigned long long)__double_as_longlong(v));
    if (prev == cur) return;
    cur = prev;
  }
}

// ---- double-double arithmetic (the variance accumulators) ----------------------------------------------------------
// A value is hi + lo with |lo| <= ulp(hi) / 2: about 106 significant bits.  The adds below are the accurate ("IEEE") variant,
// whose relative error stays near 2^-104 whatever the signs, so sums of many terms keep about 100 bits.
__device__ __forceinline__ void dd_two_sum(double a, double b, double& s, double& e) {
  s = a + b; const double bb = s - a; e = (a - (s - bb)) + (b - bb);
}
__device__ __forceinline__ void dd_fast_two_sum(double a, double b, double& s, double& e) { s = a + b; e = b - (s - a); }
__device__ __forceinline__ void dd_add(double& ah, double& al, double bh, double bl) {
  double s, e, t, f;
  dd_two_sum(ah, bh, s, e);
  dd_two_sum(al, bl, t, f);
  e += t;
  dd_fast_two_sum(s, e, s, e);
  e += f;
  dd_fast_two_sum(s, e, ah, al);
}
// n * (h + l) for an integral n below 2^53
__device__ __forceinline__ void dd_mul_d(double h, double l, double n, double& rh, double& rl) {
  const double p = h * n;
  const double e = fma(h, n, -p) + l * n;
  dd_fast_two_sum(p, e, rh, rl);
}
// one row's (or one state row's) term of a variance accumulator as a double-double: x, x^2 exactly, or, merging a state row of
// count n, mean and m2 (x = mean or m2), n * mean and m2 + n * mean^2
__device__ __forceinline__ void dd_term(int op, double x, double n, double mean, bool merging, double& h, double& l) {
  if (!merging) {
    if (op == ACC_DD_SUM) { h = x; l = 0.0; }
    else { h = x * x; l = fma(x, x, -h); }
    return;
  }
  if (op == ACC_DD_SUM) { h = n * mean; l = fma(n, mean, -h); return; }
  const double sq = mean * mean, sq_lo = fma(mean, mean, -sq);
  dd_mul_d(sq, sq_lo, n, h, l);
  dd_add(h, l, x, 0.0);
}
// 16-byte compare-and-swap loop: the table entry's double-double += (h, l)
__device__ __forceinline__ void atomic_add_dd(uint64_t* w, double h, double l) {
  if (h == 0.0 && l == 0.0) return;
  u128 cur = ((u128)w[1] << 64) | w[0];
  for (;;) {
    double ch = __longlong_as_double((long long)(uint64_t)cur), cl = __longlong_as_double((long long)(uint64_t)(cur >> 64));
    dd_add(ch, cl, h, l);
    const u128 want = ((u128)(uint64_t)__double_as_longlong(cl) << 64) | (uint64_t)__double_as_longlong(ch);
    const u128 prev = atomic_cas_128(w, cur, want);
    if (prev == cur) return;
    cur = prev;
  }
}

// identity of accumulator word `word_in_acc` (0 or 1)
__host__ __device__ inline uint64_t acc_identity(int op, int word_in_acc) {
  switch (op) {
    case ACC_MIN_I32: case ACC_MIN_I64: return 0x7FFFFFFFFFFFFFFFull;
    case ACC_MAX_I32: case ACC_MAX_I64: return 0x8000000000000000ull;
    case ACC_MIN_I128: return word_in_acc ? 0x7FFFFFFFFFFFFFFFull : 0xFFFFFFFFFFFFFFFFull;
    case ACC_MAX_I128: return word_in_acc ? 0x8000000000000000ull : 0ull;
    case ACC_MIN_F64: return 0x7FF0000000000000ull;   // +inf
    case ACC_MAX_F64: return 0xFFF0000000000000ull;   // -inf
    default: return 0ull;
  }
}
__host__ __device__ inline int acc_words_of(int op) {
  return (op == ACC_SUM_I128 || op == ACC_MIN_I128 || op == ACC_MAX_I128 || acc_is_dd(op)) ? 2 : 1;
}

// combine value into a (private or CTA-total) accumulator held in plain memory words
__device__ __forceinline__ void acc_combine_words(int op, uint64_t& w0, uint64_t& w1, uint64_t v0, uint64_t v1) {
  switch (op) {
    case ACC_SUM_I64: case ACC_COUNT: w0 += v0; break;
    case ACC_SUM_I128: { uint64_t s = w0 + v0; w1 += v1 + (s < w0 ? 1ull : 0ull); w0 = s; break; }
    case ACC_SUM_F64: w0 = (uint64_t)__double_as_longlong(__longlong_as_double((long long)w0) + __longlong_as_double((long long)v0)); break;
    case ACC_MIN_I32: case ACC_MIN_I64: if ((int64_t)v0 < (int64_t)w0) w0 = v0; break;
    case ACC_MAX_I32: case ACC_MAX_I64: if ((int64_t)v0 > (int64_t)w0) w0 = v0; break;
    case ACC_MIN_I128: { i128 a = (i128)(((u128)w1 << 64) | w0), b = (i128)(((u128)v1 << 64) | v0); if (b < a) { w0 = v0; w1 = v1; } break; }
    case ACC_MAX_I128: { i128 a = (i128)(((u128)w1 << 64) | w0), b = (i128)(((u128)v1 << 64) | v0); if (b > a) { w0 = v0; w1 = v1; } break; }
    case ACC_MIN_F64: if (__longlong_as_double((long long)v0) < __longlong_as_double((long long)w0)) w0 = v0; break;
    case ACC_MAX_F64: if (__longlong_as_double((long long)v0) > __longlong_as_double((long long)w0)) w0 = v0; break;
    case ACC_DD_SUM: case ACC_DD_SQ: {
      double h = __longlong_as_double((long long)w0), l = __longlong_as_double((long long)w1);
      dd_add(h, l, __longlong_as_double((long long)v0), __longlong_as_double((long long)v1));
      w0 = (uint64_t)__double_as_longlong(h); w1 = (uint64_t)__double_as_longlong(l);
      break;
    }
    default: break;
  }
}

__device__ __forceinline__ int64_t warp_sum_i64(int64_t v) {
#pragma unroll
  for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
  return v;
}
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
  return v;
}

// values whose magnitude is below 2^55 may be summed 128 at a time in 64 bits without overflow
__device__ __forceinline__ bool fits55(i128 v) {
  const int64_t lo = (int64_t)v;
  return (i128)lo == v && ((uint64_t)(lo + (1ll << 55)) >> 56) == 0;
}

// checked integer division: MIN / -1 and MIN % -1 have no result in T (arrow-rs div_checked / mod_checked report an
// overflow for both); a division by zero is reported as such.  Only rows that are evaluated (`live`) raise.
template <typename T> __device__ __forceinline__ T checked_div(T a, T b, bool rem, bool live, uint32_t* err) {
  const T min = (T)((u128)1 << (8 * sizeof(T) - 1));
  if (b == 0) { if (live) atomicOr(err, ERR_DIV_ZERO); return (T)0; }
  if (b == (T)-1 && a == min) { if (live) atomicOr(err, ERR_OVERFLOW); return (T)0; }
  return rem ? (T)(a % b) : (T)(a / b);
}

// a * p for a power of ten p > 1 (decimal rescale up), raising ERR_OVERFLOW for a live row whose product leaves i128.
// `lim` = I128_MAX / p; p has the factor 5, so it does not divide 2^127 and -lim is the bound below as well.
__device__ __forceinline__ i128 checked_mul_pow10(i128 a, i128 p, i128 lim, bool live, uint32_t* err) {
  if ((a > lim || a < -lim) && live) atomicOr(err, ERR_OVERFLOW);
  return (i128)((u128)a * (u128)p);
}

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

__device__ __forceinline__ uint32_t fold32(uint64_t v) { return (uint32_t)v ^ (uint32_t)(v >> 32); }

__device__ __forceinline__ unsigned long long ld_volatile_u64(const void* p) {
  unsigned long long v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// substr(view, start, count) in characters (UTF-8): the result is an inline view when it fits in 12 bytes, otherwise it
// points into the source string (a result longer than 12 bytes implies a long source, whose bytes the batch keeps alive)
__device__ __forceinline__ uint8_t view_byte(const ulonglong2& v, uint32_t i) {
  if ((uint32_t)v.x <= 12) return i < 4 ? (uint8_t)(v.x >> (32 + 8 * i)) : (uint8_t)(v.y >> (8 * (i - 4)));
  return reinterpret_cast<const uint8_t*>(v.y)[i];
}
__device__ __forceinline__ ulonglong2 view_substr(const ulonglong2& v, long long start, long long count) {
  const uint32_t n = (uint32_t)v.x;
  const long long c0 = start - 1;
  uint32_t b0 = n, b1 = n;
  long long ci = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if ((view_byte(v, i) & 0xC0) != 0x80) {          // first byte of a character
      if (ci == c0) b0 = i;
      if (count >= 0 && ci == c0 + count) { b1 = i; break; }
      ++ci;
    }
  }
  if (b0 > b1) b0 = b1;
  const uint32_t rl = b1 - b0;
  ulonglong2 r; r.x = rl; r.y = 0;
  if (rl <= 12) {
    for (uint32_t k = 0; k < rl; ++k) {
      const unsigned long long b = view_byte(v, b0 + k);
      if (k < 4) r.x |= b << (32 + 8 * k); else r.y |= b << (8 * (k - 4));
    }
  } else {
    const uint8_t* p = reinterpret_cast<const uint8_t*>(v.y) + b0;
    for (uint32_t k = 0; k < 4; ++k) r.x |= (unsigned long long)p[k] << (32 + 8 * k);
    r.y = reinterpret_cast<unsigned long long>(p);
  }
  return r;
}

// character_length(view): the bytes that are not UTF-8 continuation bytes (10xxxxxx), which for valid UTF-8 is DataFusion's
// chars().count().  A zero byte is never a continuation byte, so words loaded only in part are zero-extended.
__device__ __forceinline__ uint32_t utf8_cont_bytes(uint64_t w) { return (uint32_t)__popcll(w & ~(w << 1) & 0x8080808080808080ull); }
__device__ __forceinline__ int32_t view_char_length(const ulonglong2& v) {
  const uint32_t n = (uint32_t)v.x;
  if (n <= 12) {       // inline: bytes 0-3 in the high half of x, 4-11 in y; whatever lies past byte n is masked off
    const uint64_t hx = (v.x >> 32) & (n >= 4 ? 0xFFFFFFFFull : (1ull << (8 * n)) - 1);
    const uint64_t hy = n >= 12 ? v.y : v.y & ((1ull << (8 * (n > 4 ? n - 4 : 0))) - 1);
    return (int32_t)(n - utf8_cont_bytes(hx) - utf8_cont_bytes(hy));
  }
  // Long string: every load is naturally aligned and lies inside [p, p + n), since a batch pushed from a foreign device buffer
  // may end exactly at its last string byte.  1-, 2- and 4-byte loads reach 8-byte alignment (n >= 13 keeps them inside), one
  // 8-byte load reaches 16, 16-byte loads cover the middle and 8-, 4-, 2- and 1-byte loads the tail.
  const uint8_t* p = reinterpret_cast<const uint8_t*>(v.y);
  const uint8_t* const e = p + n;
  uint32_t c = 0;
  if (reinterpret_cast<unsigned long long>(p) & 1) { c += utf8_cont_bytes(__ldg(p)); p += 1; }
  if (reinterpret_cast<unsigned long long>(p) & 2) { c += utf8_cont_bytes(__ldg(reinterpret_cast<const unsigned short*>(p))); p += 2; }
  if (reinterpret_cast<unsigned long long>(p) & 4) { c += utf8_cont_bytes(__ldg(reinterpret_cast<const unsigned int*>(p))); p += 4; }
  if ((reinterpret_cast<unsigned long long>(p) & 8) && p + 8 <= e) { c += utf8_cont_bytes(__ldg(reinterpret_cast<const unsigned long long*>(p))); p += 8; }
  for (; p + 16 <= e; p += 16) {
    const ulonglong2 w = __ldg(reinterpret_cast<const ulonglong2*>(p));
    c += utf8_cont_bytes(w.x) + utf8_cont_bytes(w.y);
  }
  if (p + 8 <= e) { c += utf8_cont_bytes(__ldg(reinterpret_cast<const unsigned long long*>(p))); p += 8; }
  if (p + 4 <= e) { c += utf8_cont_bytes(__ldg(reinterpret_cast<const unsigned int*>(p))); p += 4; }
  if (p + 2 <= e) { c += utf8_cont_bytes(__ldg(reinterpret_cast<const unsigned short*>(p))); p += 2; }
  if (p < e) c += utf8_cont_bytes(__ldg(p));
  return (int32_t)(n - c);
}

// Order-preserving compaction of tile `tile` (tile_rows rows; thread row k is threadIdx.x + k * NT, keep[k]: it is kept), called
// by the whole CTA: returns the output position of the tile's first kept row, and at[k] = the position of kept row k within
// the tile.  warp_sums (RPT * NT / 32 words) and tile_base are the CTA's shared scratch; the caller needs a CTA barrier before
// they are written again.  The tile that ends the input writes P.out_count.
// Look-back word of P.tile_status: bits 63..62 = 0 invalid / 1 tile aggregate / 2 inclusive prefix.
template <int RPT>
__device__ __forceinline__ unsigned long long compact_positions(const PipelineParams& P, const bool (&keep)[RPT], int64_t tile, int tile_rows,
                                                                uint32_t* warp_sums, unsigned long long* tile_base, uint32_t (&at)[RPT]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, keep[k]);
    at[k] = __popc(b & ((1u << lane) - 1));
    if (lane == 0) warp_sums[k * (NT / 32) + warp] = __popc(b);
  }
  __syncthreads();
  if (warp == 0) {
    // exclusive scan of the RPT * 8 (<= 32) warp totals, in row order
    const int n = RPT * (NT / 32);
    uint32_t v = lane < n ? warp_sums[lane] : 0, incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += t; }
    if (lane < n) warp_sums[lane] = incl - v;
    const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
    // decoupled look-back, one warp wide: 32 predecessor tiles are inspected per step; the walk stops at the
    // closest tile that already published an inclusive prefix (flag 2) and adds the aggregates (flag 1) in between
    unsigned long long excl = 0;
    if (P.tile_offsets) {
      excl = P.tile_offsets[tile];             // two-pass filter: the mask pass already fixed every tile's position
    } else if (tile > 0) {
      if (lane == 0) st_release_u64(P.tile_status + tile, (1ull << 62) | total);
      int64_t hi = tile - 1;                   // newest tile not yet accounted for
      uint32_t spins = 0;
      for (;;) {
        const int64_t t = hi - lane;
        unsigned long long sw = t >= 0 ? ld_acquire_u64(P.tile_status + t) : (2ull << 62);   // before tile 0: prefix 0
        const unsigned flag = (unsigned)(sw >> 62);
        const unsigned ready = __ballot_sync(0xFFFFFFFFu, flag != 0);
        const unsigned prefix = __ballot_sync(0xFFFFFFFFu, flag == 2);
        // usable window: lanes 0..first_prefix (inclusive) if all of them are ready
        const int first_prefix = prefix ? __ffs(prefix) - 1 : 32;
        const unsigned need = first_prefix >= 31 ? 0xFFFFFFFFu : ((2u << first_prefix) - 1);
        if ((ready & need) != need) { if (++spins > (1u << 24)) __trap(); continue; }      // somebody in the window is not published yet
        unsigned long long s = (lane <= first_prefix) ? (sw & ((1ull << 62) - 1)) : 0ull;
#pragma unroll
        for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, d);
        excl += s;
        if (first_prefix < 32) break;          // reached a published prefix
        hi -= 32;
      }
    }
    if (lane == 0) {
      *tile_base = excl;
      if (!P.tile_offsets) {
        st_release_u64(P.tile_status + tile, (2ull << 62) | (excl + total));
        if ((tile + 1) * tile_rows >= P.n_rows) *P.out_count = excl + total;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < RPT; ++k) at[k] += warp_sums[k * (NT / 32) + warp];
  return *tile_base;
}

}  // namespace sg
