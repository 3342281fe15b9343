// pipeline.cu -- the fused tile-pipeline kernel (see vm.h) and its helper kernels.
//
// Replaces, in one pass over HBM, the DataFusion operator chain
//   FilterExec -> ProjectionExec -> AggregateExec(Partial|Single|Final*)      (SURVEY.md 8a a1-a3)
// that Sail drives per 8192-row batch (reference call sites: crates/sail-execution/src/
// job_runner.rs:64 `execute_stream`, crates/sail-physical-plan/src/streaming/filter.rs:104-116,
// crates/sail-plan/src/function/aggregate.rs:51-72,302-353,678-710).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "agg_hot.cuh"
#include "dev_ops.cuh"
#include "dev_util.cuh"
#include "kernels.hpp"
#include "vm.h"

namespace sg {

struct Smem {
  uint64_t full[2];        // TMA "tile landed" barriers, one per stage
  int32_t tile[2];
  uint32_t dict_n;         // groups in the CTA dictionary (agg_hot.cuh; release/acquire)
  uint32_t dict_lock;
  uint32_t cache_count;    // BUILD: occupied entries of the CTA chain cache
  int32_t defer[2];        // AGG with a bounded table: "stop taking tiles" flag, double buffered across iterations
  unsigned long long tile_base;   // COMPACT: exclusive prefix of this tile
  uint32_t warp_sums[33];
};
constexpr int SMEM_HDR = 256;

struct TileCtx {
  uint8_t* arena;
  uint32_t stage_off;      // added to stage-relative (bit 31) offsets
  int nrows;               // valid rows of this tile
  int64_t row0;
};
// offsets arrive pre-resolved per stage (KernelArgs): nothing to compute on the device
__device__ __forceinline__ uint32_t eff(const TileCtx&, uint32_t off) { return off; }

// ================================================================================================
// tile VM
// ================================================================================================
template <typename T> struct ImmOf;
template <> struct ImmOf<int32_t> { static __device__ __forceinline__ int32_t get(const VmInst& I) { return (int32_t)I.imm0; } };
template <> struct ImmOf<int64_t> { static __device__ __forceinline__ int64_t get(const VmInst& I) { return (int64_t)I.imm0; } };
template <> struct ImmOf<double> { static __device__ __forceinline__ double get(const VmInst& I) { return __longlong_as_double((long long)I.imm0); } };
template <> struct ImmOf<i128> { static __device__ __forceinline__ i128 get(const VmInst& I) { return (i128)(((u128)I.imm1 << 64) | I.imm0); } };
template <> struct ImmOf<uint8_t> { static __device__ __forceinline__ uint8_t get(const VmInst& I) { return (uint8_t)I.imm0; } };


// Operands of all RPT rows are loaded first, then computed, then stored: shared-memory loads of
// different rows may alias the stores as far as the compiler knows, so interleaving them would
// serialise the rows; batching exposes RPT independent dependency chains per instruction.
template <int RPT, typename T, bool IA, bool IB>
__device__ __forceinline__ void vm_load2(const VmInst& I, const TileCtx& c, T (&a)[RPT], T (&b)[RPT]) {
  const T imm = ImmOf<T>::get(I);
  const uint8_t* pa = c.arena + eff(c, I.a) + threadIdx.x * I.sa;
  const uint8_t* pb = c.arena + eff(c, I.b) + threadIdx.x * I.sb;
  const int sa = I.sa * NT, sb = I.sb * NT;
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    a[k] = IA ? imm : lds<T>(pa + k * sa);
    b[k] = IB ? imm : lds<T>(pb + k * sb);
  }
}
template <int RPT, typename T, typename F, bool IA, bool IB>
__device__ __forceinline__ void vm_bin_i(const VmInst& I, const TileCtx& c) {
  T a[RPT], b[RPT];
  vm_load2<RPT, T, IA, IB>(I, c, a, b);
  uint8_t* pd = c.arena + eff(c, I.dst) + threadIdx.x * (int)sizeof(T);
#pragma unroll
  for (int k = 0; k < RPT; ++k) sts<T>(pd + k * NT * (int)sizeof(T), F::template f<T>(a[k], b[k]));
}
template <int RPT, typename T, typename F>
__device__ __forceinline__ void vm_bin(const VmInst& I, const TileCtx& c) {
  if (I.flags & F_IMM_B) vm_bin_i<RPT, T, F, false, true>(I, c);
  else if (I.flags & F_IMM_A) vm_bin_i<RPT, T, F, true, false>(I, c);
  else vm_bin_i<RPT, T, F, false, false>(I, c);
}
template <int RPT, typename T, typename F, bool IA, bool IB>
__device__ __forceinline__ void vm_cmp_i(const VmInst& I, const TileCtx& c) {
  T a[RPT], b[RPT];
  vm_load2<RPT, T, IA, IB>(I, c, a, b);
  uint8_t* pd = c.arena + eff(c, I.dst) + threadIdx.x;
#pragma unroll
  for (int k = 0; k < RPT; ++k) pd[k * NT] = F::template f<T>(a[k], b[k]) ? 1 : 0;
}
template <int RPT, typename T, typename F>
__device__ __forceinline__ void vm_cmp(const VmInst& I, const TileCtx& c) {
  if (I.flags & F_IMM_B) vm_cmp_i<RPT, T, F, false, true>(I, c);
  else if (I.flags & F_IMM_A) vm_cmp_i<RPT, T, F, true, false>(I, c);
  else vm_cmp_i<RPT, T, F, false, false>(I, c);
}
template <int RPT, typename F>
__device__ __forceinline__ void vm_bin_kind(const VmInst& I, int kind, const TileCtx& c) {
  switch (kind) {
    case K_I32: vm_bin<RPT, int32_t, F>(I, c); break;
    case K_I64: vm_bin<RPT, int64_t, F>(I, c); break;
    case K_F64: vm_bin<RPT, double, F>(I, c); break;
    case K_I128: vm_bin<RPT, i128, F>(I, c); break;
    default: break;
  }
}
template <int RPT, typename F>
__device__ __forceinline__ void vm_cmp_kind(const VmInst& I, int kind, const TileCtx& c) {
  switch (kind) {
    case K_B: vm_cmp<RPT, uint8_t, F>(I, c); break;
    case K_I32: vm_cmp<RPT, int32_t, F>(I, c); break;
    case K_I64: vm_cmp<RPT, int64_t, F>(I, c); break;
    case K_F64: vm_cmp<RPT, double, F>(I, c); break;
    case K_I128: vm_cmp<RPT, i128, F>(I, c); break;
    default: break;
  }
}

// views: equality only (ordering comparisons on strings are rejected by the compiler)
template <int RPT>
__device__ __noinline__ void vm_view_eq(const VmInst& I, const TileCtx& c, bool negate) {
  const uint8_t* pa = c.arena + eff(c, I.a);
  const uint8_t* pb = c.arena + eff(c, I.b);
  uint8_t* pd = c.arena + eff(c, I.dst);
  ulonglong2 imm; imm.x = I.imm0; imm.y = I.imm1;
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    ulonglong2 a = (I.flags & F_IMM_A) ? imm : *reinterpret_cast<const ulonglong2*>(pa + r * I.sa);
    ulonglong2 b = (I.flags & F_IMM_B) ? imm : *reinterpret_cast<const ulonglong2*>(pb + r * I.sb);
    bool eq = view_equal(a, b);
    pd[r] = (eq != negate) ? 1 : 0;
  }
}

template <typename T> __device__ __forceinline__ T trunc_div(T a, T b) { return a / b; }

template <int RPT, typename T, bool REM>
__device__ __noinline__ void vm_div(const VmInst& I, const TileCtx& c, uint32_t* err) {
  const T imm = ImmOf<T>::get(I);
  const uint8_t* pa = c.arena + eff(c, I.a);
  const uint8_t* pb = c.arena + eff(c, I.b);
  const uint8_t* pg = I.c == NO_SLOT ? nullptr : c.arena + eff(c, I.c);
  uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    T a = (I.flags & F_IMM_A) ? imm : lds<T>(pa + r * I.sa);
    T b = (I.flags & F_IMM_B) ? imm : lds<T>(pb + r * I.sb);
    bool live = r < c.nrows && (pg == nullptr || pg[r]);
    sts<T>(pd + r * (int)sizeof(T), checked_div<T>(a, b, REM, live, err));
  }
}
// decimal rescale up whose product can leave i128 (compiler.cu: checked only where p + k > 38); c = rows evaluated or NO_SLOT
template <int RPT>
__device__ __noinline__ void vm_mul_pow10_checked(const VmInst& I, const TileCtx& c, uint32_t* err) {
  const i128 p = ImmOf<i128>::get(I);
  const i128 lim = (i128)(~(u128)0 >> 1) / p;
  const uint8_t* pa = c.arena + eff(c, I.a);
  const uint8_t* pg = I.c == NO_SLOT ? nullptr : c.arena + eff(c, I.c);
  uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    const bool live = r < c.nrows && (pg == nullptr || pg[r]);
    sts<i128>(pd + r * 16, checked_mul_pow10(lds<i128>(pa + r * I.sa), p, lim, live, err));
  }
}
template <int RPT>
__device__ __noinline__ void vm_div_f64(const VmInst& I, const TileCtx& c, bool rem) {
  const double imm = ImmOf<double>::get(I);
  const uint8_t* pa = c.arena + eff(c, I.a);
  const uint8_t* pb = c.arena + eff(c, I.b);
  uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    double a = (I.flags & F_IMM_A) ? imm : lds<double>(pa + r * I.sa);
    double b = (I.flags & F_IMM_B) ? imm : lds<double>(pb + r * I.sb);
    sts<double>(pd + r * 8, rem ? fmod(a, b) : a / b);
  }
}

// decimal rescale down: round half away from zero (arrow `rescale_decimal`)
template <int RPT, typename T>
__device__ __noinline__ void vm_divround(const VmInst& I, const TileCtx& c) {
  const T d = ImmOf<T>::get(I);
  const uint8_t* pa = c.arena + eff(c, I.a);
  uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    T a = lds<T>(pa + r * I.sa);
    T q = a / d, rem = a % d;
    T twice = rem < 0 ? -rem * 2 : rem * 2;
    if (twice >= d) q += (a < 0 ? -1 : 1);
    sts<T>(pd + r * (int)sizeof(T), q);
  }
}


template <int RPT>
__device__ __noinline__ void vm_cvt(const VmInst& I, int dkind, const TileCtx& c) {
  const uint8_t* pa = c.arena + eff(c, I.a);
  uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    const uint8_t* p = pa + r * I.sa;
    i128 iv = 0; double fv = 0.0; bool isf = false;
    switch (I.aux) {
      case SRC_I8: iv = lds<int8_t>(p); break;
      case SRC_I16: iv = lds<int16_t>(p); break;
      case SRC_U8: iv = lds<uint8_t>(p); break;
      case SRC_U16: iv = lds<uint16_t>(p); break;
      case SRC_U32: iv = lds<uint32_t>(p); break;
      case SRC_I32: iv = lds<int32_t>(p); break;
      case SRC_I64: iv = lds<int64_t>(p); break;
      case SRC_I128: iv = lds<i128>(p); break;
      case SRC_B: iv = lds<uint8_t>(p) ? 1 : 0; break;
      case SRC_U64: iv = (i128)lds<uint64_t>(p); break;
      case SRC_F32: fv = lds<float>(p); isf = true; break;
      case SRC_F64: fv = lds<double>(p); isf = true; break;
    }
    switch (dkind) {
      case K_I32: sts<int32_t>(pd + r * 4, isf ? (int32_t)fv : (int32_t)iv); break;
      case K_I64: sts<int64_t>(pd + r * 8, isf ? (int64_t)fv : (int64_t)iv); break;
      case K_I128: sts<i128>(pd + r * 16, isf ? (i128)(int64_t)fv : iv); break;
      case K_F64: sts<double>(pd + r * 8, isf ? fv : (I.aux == SRC_I128 || I.aux == SRC_U64 ? (double)iv : (double)(int64_t)iv)); break;
      case K_B: pd[r] = isf ? (fv != 0.0) : (iv != 0); break;
    }
  }
}

template <int RPT, typename T>
__device__ __forceinline__ void vm_select(const VmInst& I, const TileCtx& c) {
  const T imm = ImmOf<T>::get(I);
  const uint8_t* pa = c.arena + eff(c, I.a);
  const uint8_t* pb = c.arena + eff(c, I.b);
  const uint8_t* pc = c.arena + eff(c, I.c);
  uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    T a = (I.flags & F_IMM_A) ? imm : lds<T>(pa + r * I.sa);
    T b = (I.flags & F_IMM_B) ? imm : lds<T>(pb + r * I.sb);
    sts<T>(pd + r * (int)sizeof(T), pc[r] ? a : b);
  }
}
template <int RPT>
__device__ __noinline__ void vm_select_v16(const VmInst& I, const TileCtx& c) {
  const uint8_t* pa = c.arena + eff(c, I.a);
  const uint8_t* pb = c.arena + eff(c, I.b);
  const uint8_t* pc = c.arena + eff(c, I.c);
  uint8_t* pd = c.arena + eff(c, I.dst);
  ulonglong2 imm; imm.x = I.imm0; imm.y = I.imm1;
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    ulonglong2 a = (I.flags & F_IMM_A) ? imm : *reinterpret_cast<const ulonglong2*>(pa + r * I.sa);
    ulonglong2 b = (I.flags & F_IMM_B) ? imm : *reinterpret_cast<const ulonglong2*>(pb + r * I.sb);
    *reinterpret_cast<ulonglong2*>(pd + r * 16) = pc[r] ? a : b;
  }
}



template <int RPT>
__device__ __noinline__ void vm_like(const VmInst& I, const TileCtx& c) {
  const uint8_t* pa = c.arena + eff(c, I.a);
  uint8_t* pd = c.arena + eff(c, I.dst);
  const uint8_t* pat = reinterpret_cast<const uint8_t*>(I.imm1);
  const uint32_t plen = (uint32_t)I.imm0;
  const int cls = I.aux & 0xFF;
  const bool negate = (I.aux >> 8) & 1;
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    bool hit = false;
    if (r < c.nrows) {
      const uint8_t* vp = pa + r * I.sa;
      ulonglong2 v = *reinterpret_cast<const ulonglong2*>(vp);
      hit = like_match(view_ptr(v, vp), (uint32_t)v.x, pat, plen, cls);
    }
    pd[r] = (hit != negate) ? 1 : 0;
  }
}

// OP_CHAR_LEN: out of line like the other string instructions
template <int RPT>
__device__ __noinline__ void vm_char_len(const VmInst& I, const TileCtx& c) {
  const uint8_t* pa = c.arena + eff(c, I.a);
  uint8_t* pd = c.arena + eff(c, I.dst);
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    sts<int32_t>(pd + r * 4, r < c.nrows ? view_char_length(*reinterpret_cast<const ulonglong2*>(pa + r * I.sa)) : 0);
  }
}

// OP_TS_PART / OP_TS_TRUNC: out of line, so that the main VM switch keeps its registers.  The unit is chosen once per
// instruction, outside the row loop, so each loop divides by constants only.
template <int RPT, int64_t UPS, bool TRUNC>
__device__ __forceinline__ void vm_ts_rows(const VmInst& I, const TileCtx& c) {
  const uint8_t* pa = c.arena + eff(c, I.a);
  uint8_t* pd = c.arena + eff(c, I.dst);
  const int part = I.aux, kind = I.op >> 8;
  const int64_t off = (int64_t)I.imm1;
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    const int64_t v = lds<int64_t>(pa + r * I.sa);
    const int64_t x = TRUNC ? ts_trunc_u<UPS>(v, part, off) : ts_part_u<UPS>(v, part, off);
    if (kind == K_I32) sts<int32_t>(pd + r * 4, (int32_t)x);
    else sts<int64_t>(pd + r * 8, x);
  }
}
template <int RPT, bool TRUNC>
__device__ __noinline__ void vm_ts(const VmInst& I, const TileCtx& c) {
  switch (I.imm0) {
    case 1: vm_ts_rows<RPT, 1, TRUNC>(I, c); break;
    case 1000: vm_ts_rows<RPT, 1000, TRUNC>(I, c); break;
    case 1000000: vm_ts_rows<RPT, 1000000, TRUNC>(I, c); break;
    default: vm_ts_rows<RPT, 1000000000, TRUNC>(I, c);
  }
}

// ------------------------------------------------------------------------------------------------
// join probe (OP_PROBE): open-addressing lookup of the probe key in the build table
// ------------------------------------------------------------------------------------------------

// Packs the key columns of row r into 8-byte words; returns the combined hash.  *has_null is set
// when any key is NULL.  Views are kept as their 16 raw bytes (view_equal/view_hash resolve long
// strings through the absolute pointer stored by the importer).
template <int NKMAX>
__device__ __forceinline__ uint64_t pack_key(const KeyDesc* keys, int n_keys, int has_null_word, const TileCtx& c, int r,
                                             KeyRegs& k, bool* has_null) {
  uint64_t h = 0x243F6A8885A308D3ull;
  uint64_t nullmask = 0;
  int w = has_null_word ? 1 : 0;
#pragma unroll
  for (int i = 0; i < NKMAX; ++i) {
    if (i < n_keys) {
      const KeyDesc& d = keys[i];
      const uint8_t* p = c.arena + eff(c, d.slot) + r * d.stride;
      bool isnull = d.valid_slot != NO_SLOT && c.arena[eff(c, d.valid_slot) + r] == 0;
      if (isnull) nullmask |= 1ull << i;
      if (d.width == 16) {
        ulonglong2 v = *reinterpret_cast<const ulonglong2*>(p);
        if (isnull) { v.x = 0; v.y = 0; }
        k.w[w] = v.x; k.w[w + 1] = v.y;
        h = mix64(h ^ (d.is_view ? view_hash(v) : mix64(v.x ^ mix64(v.y))));
        w += 2;
      } else {
        uint64_t v = isnull ? 0 : load_key_word(p, d.width);
        k.w[w] = v;
        h = mix64(h ^ v);
        w += 1;
      }
    }
  }
  if (has_null_word) { k.w[0] = nullmask; h = mix64(h ^ nullmask); }
  *has_null = nullmask != 0;
  return h;
}

__device__ __forceinline__ bool key_words_equal(const KeyDesc* keys, int n_keys, int has_null_word, const uint64_t* a,
                                                const KeyRegs& b) {
  int w = 0;
  if (has_null_word) { if (a[0] != b.w[0]) return false; w = 1; }
  for (int i = 0; i < n_keys; ++i) {
    if (keys[i].width == 16) {
      if (keys[i].is_view) {
        ulonglong2 x, y; x.x = a[w]; x.y = a[w + 1]; y.x = b.w[w]; y.y = b.w[w + 1];
        if (!view_equal(x, y)) return false;
      } else if (a[w] != b.w[w] || a[w + 1] != b.w[w + 1]) return false;
      w += 2;
    } else {
      if (a[w] != b.w[w]) return false;
      w += 1;
    }
  }
  return true;
}

// join table slot: { u64 tag (0 = empty; hash | 1), i64 row }
// General lookup: any number / type of keys; the rows of a thread are resolved one after the other.
template <int RPT>
__device__ __noinline__ void vm_probe_general(const ProbeParams& P, const TileCtx& c, uint32_t mask_slot) {
  uint8_t* pm = c.arena + eff(c, P.match_slot);
  uint8_t* prow = c.arena + eff(c, P.rowid_slot);
  const uint8_t* pact = mask_slot == NO_SLOT ? nullptr : c.arena + eff(c, mask_slot);
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    int64_t row = -1;
    bool live = r < c.nrows && (pact == nullptr || pact[r]);
    if (live) {
      KeyRegs key; bool has_null;
      uint64_t h = pack_key<MAX_KEYS>(P.keys, P.n_keys, 0, c, r, key, &has_null);
      if (!has_null) {   // NullEqualsNothing
        uint64_t tag = h | 1ull;
        uint64_t idx = (h >> 1) & P.capacity_mask;
        for (;;) {
          const ulonglong2 s = *reinterpret_cast<const ulonglong2*>(P.table + idx * 16);
          if (s.x == 0) break;
          if (s.x == tag) {
            // verify against the build-side key columns
            const int64_t cand = (int64_t)s.y - 1;                 // slot head = row + 1
            bool eq = true;
            int w = 0;
            for (int i = 0; i < P.n_keys && eq; ++i) {
              const KeyDesc& d = P.keys[i];
              const uint8_t* bp = P.build_keys[i] + cand * P.build_stride[i];
              if (d.width == 16) {
                ulonglong2 bv = *reinterpret_cast<const ulonglong2*>(bp);
                if (d.is_view) { ulonglong2 pv; pv.x = key.w[w]; pv.y = key.w[w + 1]; eq = view_equal(bv, pv); }
                else eq = bv.x == key.w[w] && bv.y == key.w[w + 1];
                w += 2;
              } else {
                eq = load_key_word(bp, d.width) == key.w[w];
                w += 1;
              }
            }
            if (eq) { row = cand; break; }
          }
          idx = (idx + 1) & P.capacity_mask;
        }
      }
    }
    if (row >= 0 && P.visited) P.visited[row] = 1;
    pm[r] = row >= 0 ? 1 : 0;
    sts<int64_t>(prow + r * 8, row);
  }
}

// One key of at most 8 bytes (the usual integer / date join key).  The lookup is latency bound (table slot, then the
// build key of the candidate: two dependent random loads), so the RPT rows of a thread advance in lock step: all
// first-slot loads are issued together, then all candidate key loads; only rows that collide continue probing.
// Hash as pack_key(): mix64(seed ^ key word).
template <int RPT>
__device__ __noinline__ void vm_probe_narrow(const ProbeParams& P, const TileCtx& c, uint32_t mask_slot) {
  uint8_t* pm = c.arena + eff(c, P.match_slot);
  uint8_t* prow = c.arena + eff(c, P.rowid_slot);
  const uint8_t* pact = mask_slot == NO_SLOT ? nullptr : c.arena + eff(c, mask_slot);
  const KeyDesc d = P.keys[0];
  const uint8_t* pk = c.arena + eff(c, d.slot);
  const uint8_t* pv = d.valid_slot == NO_SLOT ? nullptr : c.arena + eff(c, d.valid_slot);
  const uint8_t* bcol = P.build_keys[0];
  const int bstride = P.build_stride[0];
  uint64_t key[RPT], tag[RPT], bkey[RPT];
  ulonglong2 s[RPT];
  bool act[RPT];
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    act[k] = r < c.nrows && (pact == nullptr || pact[r]) && (pv == nullptr || pv[r]);     // NULL keys match nothing
    key[k] = load_key_word(pk + r * d.stride, d.width);
    const uint64_t h = mix64(0x243F6A8885A308D3ull ^ key[k]);
    tag[k] = h | 1ull;
    s[k].x = 0; s[k].y = 0;
    if (act[k]) s[k] = *reinterpret_cast<const ulonglong2*>(P.table + ((h >> 1) & P.capacity_mask) * 16);
  }
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    bkey[k] = 0;
    if (s[k].x == tag[k]) bkey[k] = load_key_word(bcol + ((int64_t)s[k].y - 1) * bstride, d.width);      // slot head = row + 1
  }
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    int64_t row = -1;
    if (s[k].x != 0) {
      if (s[k].x == tag[k] && bkey[k] == key[k]) row = (int64_t)s[k].y - 1;
      else {                                                  // collision: ordinary linear probe from the next slot
        uint64_t idx = (((tag[k] >> 1) & P.capacity_mask) + 1) & P.capacity_mask;
        for (;;) {
          const ulonglong2 cur = *reinterpret_cast<const ulonglong2*>(P.table + idx * 16);
          if (cur.x == 0) break;
          if (cur.x == tag[k] && load_key_word(bcol + ((int64_t)cur.y - 1) * bstride, d.width) == key[k]) { row = (int64_t)cur.y - 1; break; }
          idx = (idx + 1) & P.capacity_mask;
        }
      }
    }
    if (row >= 0 && P.visited) P.visited[row] = 1;
    pm[r] = row >= 0 ? 1 : 0;
    sts<int64_t>(prow + r * 8, row);
  }
}

template <int RPT>
__device__ __forceinline__ void vm_probe(const ProbeParams& P, const TileCtx& c, uint32_t mask_slot) {
  if (P.n_keys == 1 && P.keys[0].width != 16) vm_probe_narrow<RPT>(P, c, mask_slot);
  else vm_probe_general<RPT>(P, c, mask_slot);
}

template <int RPT>
__device__ __noinline__ void vm_gather(const VmInst& I, const TileCtx& c) {
  const uint8_t* prow = c.arena + eff(c, I.a);
  uint8_t* pd = c.arena + eff(c, I.dst);
  const uint8_t* src = reinterpret_cast<const uint8_t*>(I.imm1);
  const int w = I.aux;
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    int64_t row = lds<int64_t>(prow + r * 8);
    if (w == 16) {
      ulonglong2 v; v.x = 0; v.y = 0;
      if (row >= 0) v = *reinterpret_cast<const ulonglong2*>(src + row * 16);
      *reinterpret_cast<ulonglong2*>(pd + r * 16) = v;
    } else if (w == 8) {
      sts<uint64_t>(pd + r * 8, row >= 0 ? *reinterpret_cast<const uint64_t*>(src + row * 8) : 0ull);
    } else if (w == 4) {
      sts<uint32_t>(pd + r * 4, row >= 0 ? *reinterpret_cast<const uint32_t*>(src + row * 4) : 0u);
    } else {   // bytes (validity / booleans stored one byte per row on the build side)
      pd[r] = row >= 0 ? src[row] : 0;
    }
  }
}

template <int RPT>
__device__ __noinline__ void vm_distinct_first(const AggParams& D, const TileCtx& c, uint32_t dst, uint32_t mask_slot, uint32_t* err);

template <int RPT>
__device__ __forceinline__ void vm_exec(const VmInst* prog, int n_inst, const TileCtx& c, const PipelineParams& P,
                                        const PipelineAux* aux) {
  for (int pc = 0; pc < n_inst; ++pc) {
    const VmInst& I = prog[pc];      // stays in shared memory: fields are read with uniform LDS
    const int base = I.op & 0xFF, kind = I.op >> 8;
    switch (base) {
      case OP_UNPACK_BITS: {
        const uint8_t* pa = c.arena + eff(c, I.a);
        uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          const int r = threadIdx.x + k * NT;
          pd[r] = (pa[r >> 3] >> (r & 7)) & 1;
        }
        break;
      }
      case OP_CONST: {
        uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          const int r = threadIdx.x + k * NT;
          switch (kind) {
            case K_B: pd[r] = (uint8_t)I.imm0; break;
            case K_I32: sts<int32_t>(pd + r * 4, (int32_t)I.imm0); break;
            case K_I64: case K_F64: sts<uint64_t>(pd + r * 8, I.imm0); break;
            default: { ulonglong2 v; v.x = I.imm0; v.y = I.imm1; *reinterpret_cast<ulonglong2*>(pd + r * 16) = v; }
          }
        }
        break;
      }
      case OP_MOV: {
        const uint8_t* pa = c.arena + eff(c, I.a);
        uint8_t* pd = c.arena + eff(c, I.dst);
        const int w = kind_width(kind);
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          const int r = threadIdx.x + k * NT;
          if (w == 16) *reinterpret_cast<ulonglong2*>(pd + r * 16) = *reinterpret_cast<const ulonglong2*>(pa + r * I.sa);
          else if (w == 8) sts<uint64_t>(pd + r * 8, lds<uint64_t>(pa + r * I.sa));
          else if (w == 4) sts<uint32_t>(pd + r * 4, lds<uint32_t>(pa + r * I.sa));
          else pd[r] = pa[r * I.sa];
        }
        break;
      }
      case OP_CVT: vm_cvt<RPT>(I, kind, c); break;
      case OP_ADD: vm_bin_kind<RPT, OpAdd>(I, kind, c); break;
      case OP_SUB: vm_bin_kind<RPT, OpSub>(I, kind, c); break;
      case OP_MUL: vm_bin_kind<RPT, OpMul>(I, kind, c); break;
      case OP_DIV:
      case OP_REM:
        if (kind == K_F64) vm_div_f64<RPT>(I, c, base == OP_REM);
        else if (kind == K_I32) { if (base == OP_DIV) vm_div<RPT, int32_t, false>(I, c, P.error_flag); else vm_div<RPT, int32_t, true>(I, c, P.error_flag); }
        else if (kind == K_I64) { if (base == OP_DIV) vm_div<RPT, int64_t, false>(I, c, P.error_flag); else vm_div<RPT, int64_t, true>(I, c, P.error_flag); }
        else { if (base == OP_DIV) vm_div<RPT, i128, false>(I, c, P.error_flag); else vm_div<RPT, i128, true>(I, c, P.error_flag); }
        break;
      case OP_NEG: {
        const uint8_t* pa = c.arena + eff(c, I.a);
        uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          const int r = threadIdx.x + k * NT;
          switch (kind) {
            case K_I32: sts<int32_t>(pd + r * 4, (int32_t)(0u - (uint32_t)lds<int32_t>(pa + r * I.sa))); break;
            case K_I64: sts<int64_t>(pd + r * 8, (int64_t)(0ull - (uint64_t)lds<int64_t>(pa + r * I.sa))); break;
            case K_F64: sts<double>(pd + r * 8, -lds<double>(pa + r * I.sa)); break;
            default: sts<i128>(pd + r * 16, (i128)((u128)0 - (u128)lds<i128>(pa + r * I.sa)));
          }
        }
        break;
      }
      case OP_MULW: {
        int64_t a[RPT], b[RPT];
        if (I.flags & F_IMM_B) vm_load2<RPT, int64_t, false, true>(I, c, a, b);
        else if (I.flags & F_IMM_A) vm_load2<RPT, int64_t, true, false>(I, c, a, b);
        else vm_load2<RPT, int64_t, false, false>(I, c, a, b);
        uint8_t* pd = c.arena + eff(c, I.dst) + threadIdx.x * 16;
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          ulonglong2 w;
          w.x = (unsigned long long)a[k] * (unsigned long long)b[k];
          w.y = (unsigned long long)__mul64hi((long long)a[k], (long long)b[k]);
          *reinterpret_cast<ulonglong2*>(pd + k * NT * 16) = w;
        }
        break;
      }
      case OP_MUL128_64: {
        const int64_t imm = (int64_t)I.imm0;
        const uint8_t* pa = c.arena + eff(c, I.a) + threadIdx.x * I.sa;
        const uint8_t* pb = c.arena + eff(c, I.b) + threadIdx.x * I.sb;
        uint8_t* pd = c.arena + eff(c, I.dst) + threadIdx.x * 16;
        ulonglong2 a[RPT]; int64_t b[RPT];
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          a[k] = *reinterpret_cast<const ulonglong2*>(pa + k * NT * I.sa);
          b[k] = (I.flags & F_IMM_B) ? imm : lds<int64_t>(pb + k * NT * I.sb);
        }
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          // (ahi:alo) * sext(b)  mod 2^128
          const unsigned long long ub = (unsigned long long)b[k];
          ulonglong2 w;
          w.x = a[k].x * ub;
          w.y = __umul64hi(a[k].x, ub) + a[k].y * ub - (b[k] < 0 ? a[k].x : 0ull);
          *reinterpret_cast<ulonglong2*>(pd + k * NT * 16) = w;
        }
        break;
      }
      case OP_DIVROUND:
        if (kind == K_I64) vm_divround<RPT, int64_t>(I, c); else vm_divround<RPT, i128>(I, c);
        break;
      case OP_MUL_POW10_CHK: vm_mul_pow10_checked<RPT>(I, c, P.error_flag); break;
      case OP_EQ: if (kind == K_V16) vm_view_eq<RPT>(I, c, false); else vm_cmp_kind<RPT, CmpEq>(I, kind, c); break;
      case OP_NE: if (kind == K_V16) vm_view_eq<RPT>(I, c, true); else vm_cmp_kind<RPT, CmpNe>(I, kind, c); break;
      case OP_LT: vm_cmp_kind<RPT, CmpLt>(I, kind, c); break;
      case OP_LE: vm_cmp_kind<RPT, CmpLe>(I, kind, c); break;
      case OP_GT: vm_cmp_kind<RPT, CmpGt>(I, kind, c); break;
      case OP_GE: vm_cmp_kind<RPT, CmpGe>(I, kind, c); break;
      case OP_AND: case OP_OR: case OP_ANDNOT: case OP_NOT: {
        const uint8_t* pa = c.arena + eff(c, I.a);
        const uint8_t* pb = c.arena + eff(c, I.b);
        uint8_t* pd = c.arena + eff(c, I.dst);
        const uint8_t imm = (uint8_t)I.imm0;
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          const int r = threadIdx.x + k * NT;
          uint8_t a = (I.flags & F_IMM_A) ? imm : pa[r];
          uint8_t b = (base == OP_NOT) ? 0 : ((I.flags & F_IMM_B) ? imm : pb[r]);
          uint8_t v = base == OP_AND ? (a & b) : base == OP_OR ? (a | b) : base == OP_ANDNOT ? (a & (b ^ 1)) : (a ^ 1);
          pd[r] = v & 1;
        }
        break;
      }
      case OP_SELECT:
        switch (kind) {
          case K_B: vm_select<RPT, uint8_t>(I, c); break;
          case K_I32: vm_select<RPT, int32_t>(I, c); break;
          case K_I64: vm_select<RPT, int64_t>(I, c); break;
          case K_F64: vm_select<RPT, double>(I, c); break;
          case K_I128: vm_select<RPT, i128>(I, c); break;
          default: vm_select_v16<RPT>(I, c);
        }
        break;
      case OP_STR_EQ_LONG: {
        // literal longer than 12 bytes: imm0 = len | prefix << 32, imm1 = device pointer to the bytes
        ulonglong2 lit; lit.x = I.imm0; lit.y = I.imm1;
        const uint8_t* pa = c.arena + eff(c, I.a);
        uint8_t* pd = c.arena + eff(c, I.dst);
        for (int k = 0; k < RPT; ++k) {
          const int r = threadIdx.x + k * NT;
          ulonglong2 a = *reinterpret_cast<const ulonglong2*>(pa + r * I.sa);
          bool eq = r < c.nrows && view_equal(a, lit);
          pd[r] = (eq != (bool)(I.aux & 1)) ? 1 : 0;
        }
        break;
      }
      case OP_STR_LIKE: vm_like<RPT>(I, c); break;
      case OP_DATE_PART: {
        const uint8_t* pa = c.arena + eff(c, I.a);
        uint8_t* pd = c.arena + eff(c, I.dst);
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          const int r = threadIdx.x + k * NT;
          int y, m, d;
          civil_from_days(lds<int32_t>(pa + r * I.sa), y, m, d);
          sts<int32_t>(pd + r * 4, I.aux == 0 ? y : I.aux == 1 ? m : d);
        }
        break;
      }
      case OP_SUBSTR: {
        const uint8_t* pa = c.arena + eff(c, I.a);
        uint8_t* pd = c.arena + eff(c, I.dst);
        for (int k = 0; k < RPT; ++k) {
          const int r = threadIdx.x + k * NT;
          ulonglong2 v; v.x = 0; v.y = 0;
          if (r < c.nrows) v = view_substr(*reinterpret_cast<const ulonglong2*>(pa + r * I.sa), (long long)I.imm0, (long long)I.imm1);
          *reinterpret_cast<ulonglong2*>(pd + r * 16) = v;
        }
        break;
      }
      case OP_CHAR_LEN: vm_char_len<RPT>(I, c); break;
      case OP_TS_PART: vm_ts<RPT, false>(I, c); break;
      case OP_TS_TRUNC: vm_ts<RPT, true>(I, c); break;
      case OP_PROBE: vm_probe<RPT>(aux->probe[I.aux], c, I.c); break;
      case OP_GATHER: vm_gather<RPT>(I, c); break;
      case OP_DISTINCT_FIRST: vm_distinct_first<RPT>(aux->distinct[I.aux], c, I.dst, I.c, P.error_flag); break;
      default: break;
    }
  }
}

// ================================================================================================
// tile loading
// ================================================================================================
__device__ __forceinline__ uint32_t tile_bytes_of(const InputCol& in, int tile_rows) {
  return in.width ? (uint32_t)in.width * tile_rows : (uint32_t)(tile_rows >> 3);
}

// cooperative copy (partial / unaligned tiles): zero-fills rows >= nrows
__device__ __forceinline__ void load_tile_generic(const PipelineParams& P, uint8_t* arena, int64_t row0, int nrows) {
  for (int i = 0; i < P.n_inputs; ++i) {
    const InputCol& in = P.in[i];
    uint8_t* dst = arena + in.slot;
    const uint32_t total = tile_bytes_of(in, P.tile_rows);
    const uint32_t valid = in.width ? (uint32_t)in.width * nrows : (uint32_t)((nrows + 7) >> 3);
    const uint8_t* src = in.data + (in.width ? (int64_t)in.width * row0 : (row0 >> 3));
    if (in.tma_ok && (valid & 15u) == 0) {
      for (uint32_t o = threadIdx.x * 16; o < total; o += NT * 16) {
        uint4 v = make_uint4(0, 0, 0, 0);
        if (o < valid) v = *reinterpret_cast<const uint4*>(src + o);
        *reinterpret_cast<uint4*>(dst + o) = v;
      }
    } else {
      for (uint32_t o = threadIdx.x; o < total; o += NT) dst[o] = o < valid ? src[o] : 0;
    }
  }
}

// ================================================================================================
// aggregation: global table
// ================================================================================================


// The interpreter's arguments to the group-table functions of agg_hot.cuh: identities from the accumulator descriptors, keys
// compared by the key descriptors.
__device__ __forceinline__ auto agg_init() {
  return [](const AggParams& A, uint64_t* acc) {
    for (int j = 0; j < A.n_accs; ++j)
      for (int w = 0; w < acc_words_of(A.accs[j].op); ++w) acc[A.accs[j].word + w] = acc_identity(A.accs[j].op, w);
  };
}
__device__ __forceinline__ auto agg_eq() {
  return [](const AggParams& A, const uint64_t* k, const KeyRegs& key) { return key_words_equal(A.keys, A.n_keys, A.has_null_word, k, key); };
}

// OP_DISTINCT_FIRST: the gate of a DISTINCT aggregate.  Every active row with a valid argument looks its (group key, argument)
// pair up in the pair set D (key: null-mask word, group keys, argument last); the row whose lookup inserted the pair passes.
// The set is never emptied, so over the whole input exactly one row per pair passes, and the accumulators behind the gate
// see every distinct argument of a group once.  Rows of one warp with the same pair share one lookup (the warp front end).
template <int RPT>
__device__ __noinline__ void vm_distinct_first(const AggParams& D, const TileCtx& c, uint32_t dst, uint32_t mask_slot, uint32_t* err) {
  uint8_t* pd = c.arena + eff(c, dst);
  const uint8_t* pact = mask_slot == NO_SLOT ? nullptr : c.arena + eff(c, mask_slot);
  const uint32_t xv = D.keys[D.n_keys - 1].valid_slot;
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    const bool live = r < c.nrows && (pact == nullptr || pact[r]) && (xv == NO_SLOT || c.arena[eff(c, xv) + r]);
    KeyRegs key; bool hn; uint64_t h = 0;
    if (live) h = pack_key<MAX_KEYS>(D.keys, D.n_keys, 1, c, r, key, &hn);
    bool first = false;
    find_or_insert_warp<FROM_A, FROM_A>(D, key, h, live, err, agg_init(), agg_eq(), &first);
    pd[r] = first ? 1 : 0;
  }
}

// hash of an already packed key (same value pack_key() returns for the row it was packed from)
__device__ __forceinline__ uint64_t hash_packed_key(const AggParams& A, const KeyRegs& key) {
  uint64_t h = 0x243F6A8885A308D3ull;
  int w = A.has_null_word ? 1 : 0;
  for (int i = 0; i < A.n_keys; ++i) {
    if (A.keys[i].width == 16) {
      ulonglong2 v; v.x = key.w[w]; v.y = key.w[w + 1];
      h = mix64(h ^ (A.keys[i].is_view ? view_hash(v) : mix64(v.x ^ mix64(v.y))));
      w += 2;
    } else { h = mix64(h ^ key.w[w]); w += 1; }
  }
  if (A.has_null_word) h = mix64(h ^ key.w[0]);
  return h;
}


// a variance accumulator's term travels as a double-double: high part in f, low part in the low word of i
__device__ __forceinline__ void set_dd_value(AccVal& v, int op, double x, double n, double mean, bool merging) {
  double h, l;
  dd_term(op, x, n, mean, merging, h, l);
  v.f = h; v.i = (i128)(uint64_t)__double_as_longlong(l);
}
__device__ __forceinline__ AccVal load_acc_value(const AccDesc& d, const TileCtx& c, int r) {
  AccVal v; v.i = 0; v.f = 0.0; v.valid = true;
  if (d.valid_slot != NO_SLOT) v.valid = c.arena[eff(c, d.valid_slot) + r] != 0;
  if (d.value_slot == NO_SLOT) return v;
  const uint8_t* p = c.arena + eff(c, d.value_slot) + r * d.stride;
  switch (d.vkind) {
    case K_I32: v.i = lds<int32_t>(p); break;
    case K_I64: v.i = lds<int64_t>(p); break;
    case K_I128: v.i = lds<i128>(p); break;
    case K_F64: v.f = lds<double>(p); break;
    case K_B: v.i = *p; break;
    default: break;
  }
  if (acc_is_dd(d.op)) {
    const bool merging = d.n_slot != NO_SLOT;
    const double n = merging ? lds<double>(c.arena + eff(c, d.n_slot) + r * 8) : 0.0;
    const double mean = merging ? lds<double>(c.arena + eff(c, d.mean_slot) + r * 8) : 0.0;
    set_dd_value(v, d.op, v.f, n, mean, merging);
  }
  return v;
}


// packed key of row r as 8-byte words held in registers (static indexing), padded with zeros to HOT_KEY_WORDS
__device__ __forceinline__ void pack_words(const AggParams& A, const TileCtx& c, int r, HotKey& kw) {
  uint64_t nullmask = 0;
#pragma unroll
  for (int w = 0; w < HOT_KEY_WORDS; ++w) {
    kw.w[w] = 0;
    if (w < A.key_words && !(A.has_null_word && w == 0)) {
      const KeyWord& d = A.kwords[w];
      const uint8_t* p = c.arena + d.slot + r * d.stride + d.byte_off;
      uint64_t v = d.width == 8 ? lds<uint64_t>(p) : d.width == 4 ? (uint64_t)lds<uint32_t>(p) : (uint64_t)*p;
      if (d.valid_slot != NO_SLOT && c.arena[d.valid_slot + r] == 0) { v = 0; nullmask |= 1ull << d.key_index; }
      kw.w[w] = v;
    }
  }
  if (A.has_null_word) kw.w[0] = nullmask;
}

// dictionary key of row r: every key word is a plain 8-byte load (views, int64, decimals) unless the plan has narrow or
// nullable keys, in which case the general packer runs
__device__ __forceinline__ void reg_pack(const AggParams& A, const TileCtx& c, int r, HotKey& kw) {
  if (A.kw_simple) {
#pragma unroll
    for (int w = 0; w < HOT_KEY_WORDS; ++w)
      kw.w[w] = w < A.key_words ? lds<uint64_t>(c.arena + A.kwords[w].slot + r * A.kwords[w].stride + A.kwords[w].byte_off) : 0ull;
  } else {
    pack_words(A, c, r, kw);
  }
}

__device__ __forceinline__ HotDict hot_dict(const AggParams& A, uint8_t* arena) { return hot_dict(arena + A.hot_smem_off, A.hot_groups); }

// entry_of(g): the table entry of dictionary group g (agg_hot.cuh: hot_entry)
__device__ __forceinline__ auto agg_entry_of(const PipelineParams& P, const AggParams& A, const HotDict& H) {
  return [&P, &A, H](int g) {
    return hot_entry<FROM_A, FROM_A, KeyRegs>(H, g, A, P.error_flag,
                              [](const AggParams& T, const KeyRegs& k) { return hash_packed_key(T, k); }, agg_init(), agg_eq());
  };
}

// rows whose group is not in the CTA-local dictionary: global table, one warp-cooperative lookup per row slot

template <int RPT>
__device__ __noinline__ void agg_cold_rows(const PipelineParams& P, const AggParams& A, const TileCtx& c, const int (&gid)[RPT], const bool (&live)[RPT]) {
  // the table walk below is a chain of dependent global accesses per row: start the first state word and entry line of
  // every row of this thread on their way first
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    if (live[k] && gid[k] < 0) {
      KeyRegs key; bool hn;
      const uint64_t h = pack_key<MAX_KEYS>(A.keys, A.n_keys, A.has_null_word, c, threadIdx.x + k * NT, key, &hn);
      const uint64_t idx = h & A.capacity_mask;
      prefetch_l2(A.state + idx);
      prefetch_l2(reinterpret_cast<const uint64_t*>(A.table) + idx * A.entry_words);
    }
  }
  for (int k = 0; k < RPT; ++k) {
    const bool cold = live[k] && gid[k] < 0;
    if (__any_sync(0xFFFFFFFFu, cold)) {
      const int r = threadIdx.x + k * NT;
      KeyRegs key; bool hn; uint64_t h = 0;
      if (cold) h = pack_key<MAX_KEYS>(A.keys, A.n_keys, A.has_null_word, c, r, key, &hn);
      uint64_t* e = find_or_insert_warp<FROM_A, FROM_A>(A, key, h, cold, P.error_flag, agg_init(), agg_eq());
      if (cold && e) {
        for (int j = 0; j < A.n_accs; ++j) {
          const AccDesc& d = A.accs[j];
          acc_global(e, A.key_words, d.op, d.word, j, d.track_seen != 0, load_acc_value(d, c, r));
        }
      }
    }
  }
}

// high-cardinality variant (AggParams::cold_only): no dictionary, every live row goes to the global table
template <int RPT>
__device__ __forceinline__ void sink_agg_cold(const PipelineParams& P, const AggParams& A, const TileCtx& c) {
  const uint8_t* pact = P.mask_slot == NO_SLOT ? nullptr : c.arena + P.mask_slot;
  int gid[RPT];
  bool live[RPT];
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    live[k] = r < c.nrows && (pact == nullptr || pact[r]);
    gid[k] = -1;
  }
  agg_cold_rows<RPT>(P, A, c, gid, live);
}

// Low-cardinality grouping (TPC-H Q1: 4 groups): every row finds its group in the CTA dictionary (agg_hot.cuh); then,
// accumulator by accumulator and group by group, the warp reduces its rows with shuffles and lane 0 folds the warp total into
// the warp's accumulator block.  No atomics, no per-thread state, ~G*n_accs*30 instructions per warp-tile regardless of tile size.
template <int RPT>
__device__ __forceinline__ void sink_agg(const PipelineParams& P, const AggParams& A, const TileCtx& c, Smem* sm) {
  const uint8_t* pact = P.mask_slot == NO_SLOT ? nullptr : c.arena + P.mask_slot;
  const HotDict H = hot_dict(A, c.arena);
  int gid[RPT];
  bool live[RPT];
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    live[k] = r < c.nrows && (pact == nullptr || pact[r]);
    gid[k] = -1;
  }
  if (A.hot_groups > 0) {
    hot_assign<HOT_MAX_GROUPS>(H, &sm->dict_n, &sm->dict_lock, A.hot_groups, live, gid,
                               [&](int k, HotKey& kw) { reg_pack(A, c, threadIdx.x + k * NT, kw); });
    const int hot_n = __shfl_sync(0xFFFFFFFFu, (int)lds_acquire_u32(&sm->dict_n), 0);      // every gid of this warp is below it
    bool anyhot = false;
#pragma unroll
    for (int k = 0; k < RPT; ++k) anyhot |= gid[k] >= 0;
    if (__any_sync(0xFFFFFFFFu, anyhot)) {
      for (int j = 0; j < A.n_accs; ++j) {
        const AccDesc& d = A.accs[j];
        AccVal av[RPT];
#pragma unroll
        for (int k = 0; k < RPT; ++k) {
          av[k].i = 0; av[k].f = 0.0; av[k].valid = false;
          if (gid[k] >= 0) av[k] = load_acc_value(d, c, threadIdx.x + k * NT);
        }
        hot_fold<RPT>(H, A.hot_groups, A.n_accs, hot_n, A.key_words, d.op, d.word, j, d.track_seen != 0, av, gid, agg_entry_of(P, A, H));
      }
    }
  }
  {
    bool anycold = false;
#pragma unroll
    for (int k = 0; k < RPT; ++k) anycold |= live[k] && gid[k] < 0;
    if (__any_sync(0xFFFFFFFFu, anycold)) agg_cold_rows<RPT>(P, A, c, gid, live);   // warp-level: no CTA barrier
  }
}

// ---- integer fast path: register-resident partials (agg_hot.cuh: RegAcc) ------------------------------------------------
// R.v[g][j]: this thread's running 64-bit partial of accumulator j for hot group g.
template <int RPT>
__device__ __forceinline__ void sink_agg_reg(const PipelineParams& P, const AggParams& A, const TileCtx& c, Smem* sm, RegAcc<REG_ACCS>& R) {
  const uint8_t* pact = P.mask_slot == NO_SLOT ? nullptr : c.arena + P.mask_slot;
  const HotDict H = hot_dict(A, c.arena);
  int gid[RPT];
  bool live[RPT];
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    live[k] = r < c.nrows && (pact == nullptr || pact[r]);
  }
  hot_assign<REG_GROUPS>(H, &sm->dict_n, &sm->dict_lock, REG_GROUPS, live, gid,
                         [&](int k, HotKey& kw) { reg_pack(A, c, threadIdx.x + k * NT, kw); });
  // accumulate: values first (RPT x n_accs loads), then predicated adds into the register partials
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    const bool hot = live[k] && gid[k] >= 0;
    if (hot) {
      int64_t val[REG_ACCS];
#pragma unroll
      for (int j = 0; j < REG_ACCS; ++j) {
        val[j] = 0;
        if (j < A.n_accs) {
          const AggParams::RegLoad& L = A.rload[j];          // constant bank, static index
          if (L.mode == 0) val[j] = 1;
          else {
            const uint8_t* p = c.arena + L.slot + r * L.stride;
            if (L.mode == 3) { val[j] = lds<int64_t>(p); continue; }         // statically below 2^55: no check
            i128 x;
            if (L.mode == 1) x = (i128)lds<int64_t>(p); else x = lds<i128>(p);
            if (fits55(x)) val[j] = (int64_t)x;
            else {                                            // rare: exact value straight to the table entry
              uint64_t* e = agg_entry_of(P, A, H)(gid[k]);
              // (an Int64 sum has one word and is defined mod 2^64: no carry into the next accumulator)
              if (e) acc_apply(A.accs[j].op, e + 2 + A.key_words + A.accs[j].word, i128_lo(x), i128_hi(x));
            }
          }
        }
      }
      reg_add(R, gid[k], val);
    }
  }
  R.rows += RPT;
  if (R.rows >= REG_FLUSH) reg_flush(H, A.n_accs, R);
  {
    bool anycold = false;
#pragma unroll
    for (int k = 0; k < RPT; ++k) anycold |= live[k] && gid[k] < 0;
    if (__any_sync(0xFFFFFFFFu, anycold)) agg_cold_rows<RPT>(P, A, c, gid, live);   // warp-level: no CTA barrier
  }
}

// ================================================================================================
// store / compact sinks
// ================================================================================================
__device__ __forceinline__ void store_value(const OutputCol& o, const TileCtx& c, int r, int64_t pos) {
  const uint8_t* p = c.arena + eff(c, o.slot) + r * o.stride;
  uint8_t* dst = o.data + pos * o.width;
  // (slot stride, output width): 16->16 copy, 8->16 sign-extend (narrow decimal), 8->8, 4->4, 4->1/2 truncate, 8->4
  if (o.width == 16) {
    if (o.stride >= 16) *reinterpret_cast<ulonglong2*>(dst) = *reinterpret_cast<const ulonglong2*>(p);
    else { int64_t v = lds<int64_t>(p); ulonglong2 w; w.x = (unsigned long long)v; w.y = (unsigned long long)(v >> 63); *reinterpret_cast<ulonglong2*>(dst) = w; }
  } else if (o.width == 8) {
    *reinterpret_cast<uint64_t*>(dst) = lds<uint64_t>(p);
  } else if (o.width == 4) {
    *reinterpret_cast<uint32_t*>(dst) = lds<uint32_t>(p);
  } else if (o.width == 2) {
    *reinterpret_cast<uint16_t*>(dst) = (uint16_t)lds<uint32_t>(p);
  } else {
    *dst = *p;
  }
}

template <int RPT>
__device__ __forceinline__ void sink_store(const PipelineParams& P, const TileCtx& c) {
  const int lane = threadIdx.x & 31;
  for (int j = 0; j < P.n_out; ++j) {
    const OutputCol& o = P.out[j];
#pragma unroll
    for (int k = 0; k < RPT; ++k) {
      const int r = threadIdx.x + k * NT;
      const bool in = r < c.nrows;
      if (o.width) { if (in) store_value(o, c, r, c.row0 + r); }
      else {   // boolean column -> bitmap word per 32 rows
        const uint32_t bits = __ballot_sync(0xFFFFFFFFu, in && c.arena[eff(c, o.slot) + r]);
        if (lane == 0 && (r - lane) < c.nrows) reinterpret_cast<uint32_t*>(o.data)[(c.row0 + r) >> 5] = bits;
      }
      if (o.valid_slot != NO_SLOT) {
        const uint32_t vb = __ballot_sync(0xFFFFFFFFu, in && c.arena[eff(c, o.valid_slot) + r]);
        if (lane == 0 && (r - lane) < c.nrows) reinterpret_cast<uint32_t*>(o.valid_bytes)[(c.row0 + r) >> 5] = vb;
      }
    }
  }
}

template <int RPT>
__device__ __forceinline__ void sink_compact(const PipelineParams& P, const TileCtx& c, Smem* sm, int64_t tile) {
  const uint8_t* pact = P.mask_slot == NO_SLOT ? nullptr : c.arena + eff(c, P.mask_slot);
  bool keep[RPT];
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    keep[k] = r < c.nrows && (pact == nullptr || pact[r]);
  }
  uint32_t at[RPT];
  const unsigned long long base = compact_positions<RPT>(P, keep, tile, P.tile_rows, sm->warp_sums, &sm->tile_base, at);
  for (int j = 0; j < P.n_out; ++j) {
    const OutputCol& o = P.out[j];
#pragma unroll
    for (int k = 0; k < RPT; ++k) {
      if (!keep[k]) continue;
      const int r = threadIdx.x + k * NT;
      const int64_t pos = (int64_t)(base + at[k]);
      if (o.width) store_value(o, c, r, pos);
      else o.data[pos] = c.arena[eff(c, o.slot) + r];                  // boolean column as bytes (packed later)
      if (o.valid_slot != NO_SLOT) o.valid_bytes[pos] = c.arena[eff(c, o.valid_slot) + r];
    }
  }
}

// ================================================================================================
// join build sink / partition sink
// ================================================================================================
// does build row `cand` carry the key packed in `key`?
__device__ __forceinline__ bool build_row_has_key(const KeyDesc* keys, const uint8_t* const* cols, const uint8_t* strides, int n_keys,
                                                  int64_t cand, const KeyRegs& key) {
  int w = 0;
  for (int i = 0; i < n_keys; ++i) {
    const KeyDesc& d = keys[i];
    const uint8_t* bp = cols[i] + cand * strides[i];
    if (d.width == 16) {
      ulonglong2 bv = *reinterpret_cast<const ulonglong2*>(bp);
      if (d.is_view) { ulonglong2 pv; pv.x = key.w[w]; pv.y = key.w[w + 1]; if (!view_equal(bv, pv)) return false; }
      else if (bv.x != key.w[w] || bv.y != key.w[w + 1]) return false;
      w += 2;
    } else {
      if (load_key_word(bp, d.width) != key.w[w]) return false;
      w += 1;
    }
  }
  return true;
}

// Join table slot = { u64 tag (0 = empty; hash | 1), u64 head (row + 1 of the newest row with this key; 0 = none yet) }.
// The tag is claimed once with a 64-bit CAS and never changes; rows are pushed on the slot's stack with ONE atomic
// exchange of `head` (wait-free: no retry loop, so a build side with a handful of distinct keys does not collapse into
// CAS retries), and next[] links them.  The probe runs in a later launch and reads slots with plain loads.
__device__ __forceinline__ void chain_push(const BuildParams& B, uint8_t* slot, long long first, long long last) {
  const unsigned long long prev = atomicExch(reinterpret_cast<unsigned long long*>(slot + 8), (unsigned long long)(first + 1));
  B.next[last] = (long long)prev - 1;                            // -1 ends the chain
  if ((prev != 0 || first != last) && *reinterpret_cast<volatile uint32_t*>(B.dup_flag) == 0) atomicOr(B.dup_flag, 1u);
}
// Finds the slot of `key`, claiming an empty one if the key is new.  A claimer publishes its pre-linked chain first..last
// at once (*pushed = true) so that later arrivals can verify their key against a row of the chain; for an existing key
// the slot is returned and the caller decides where to push (CTA chain cache or the slot itself).  nullptr: table full.
__device__ __forceinline__ uint8_t* build_find_or_claim(const BuildParams& B, const KeyRegs& key, uint64_t h, long long first, long long last, bool* pushed) {
  const unsigned long long tag = h | 1ull;
  uint64_t idx = (h >> 1) & B.capacity_mask;
  *pushed = false;
  for (uint64_t probes = 0; probes <= B.capacity_mask; ++probes) {
    uint8_t* slot = B.table + idx * 16;
    unsigned long long t = ld_volatile_u64(slot);
    if (t == 0ull) {
      t = atomicCAS(reinterpret_cast<unsigned long long*>(slot), 0ull, tag);
      if (t == 0ull) { chain_push(B, slot, first, last); *pushed = true; return slot; }      // claimed an empty slot
    }
    if (t == tag) {
      // same tag: compare with a row that is already on the chain (the claimer publishes its rows right after the CAS)
      unsigned long long head = ld_volatile_u64(slot + 8);
      for (uint32_t spins = 0; head == 0ull; ++spins) {
        if (spins > (1u << 24)) __trap();
        __nanosleep(20);
        head = ld_volatile_u64(slot + 8);
      }
      if (build_row_has_key(B.keys, B.key_cols, B.key_stride, B.n_keys, (int64_t)head - 1, key)) return slot;
    }
    idx = (idx + 1) & B.capacity_mask;
  }
  return nullptr;
}

// CTA chain cache (shared memory, lives for the whole kernel): chains for keys that already own a slot are collected
// per CTA and pushed on the slot once -- at the end of the kernel, or when the cache runs full.  A build side with a
// handful of distinct keys (a fact-like intermediate joined to a dimension: TPC-H Q5 / Q7 shapes) otherwise funnels
// millions of atomic exchanges into a few addresses.
struct ChainCacheEntry { unsigned long long slot, first; long long last; };
constexpr int CHAIN_CACHE_ENTRIES = 512;
__device__ __forceinline__ bool chain_cache_push(const BuildParams& B, ChainCacheEntry* cache, uint32_t* count, uint8_t* slot, long long first, long long last) {
  const unsigned long long sp = reinterpret_cast<unsigned long long>(slot);
  uint32_t idx = (uint32_t)mix64(sp) & (CHAIN_CACHE_ENTRIES - 1);
  for (int probe = 0; probe < 8; ++probe) {
    ChainCacheEntry* e = cache + idx;
    const unsigned long long s = atomicCAS(&e->slot, 0ull, sp);
    if (s == 0ull) atomicAdd(count, 1u);
    if (s == 0ull || s == sp) {
      const unsigned long long prev = atomicExch(&e->first, (unsigned long long)(first + 1));
      if (prev == 0ull) e->last = last;                  // this chain is the bottom of the cached stack
      else B.next[last] = (long long)prev - 1;
      return true;
    }
    idx = (idx + 1) & (CHAIN_CACHE_ENTRIES - 1);
  }
  return false;
}
// all threads of the CTA; ends with a barrier
__device__ __forceinline__ void chain_cache_flush(const BuildParams& B, ChainCacheEntry* cache, uint32_t* count) {
  __syncthreads();
  for (int i = threadIdx.x; i < CHAIN_CACHE_ENTRIES; i += NT) {
    ChainCacheEntry* e = cache + i;
    if (e->slot) {
      chain_push(B, reinterpret_cast<uint8_t*>(e->slot), (long long)e->first - 1, e->last);
      e->slot = 0ull; e->first = 0ull;
    }
  }
  if (threadIdx.x == 0) *count = 0;
  __syncthreads();
}

// HashJoinExec build: one slot per DISTINCT key; rows with an equal key are pushed on the slot's chain (next[]).
// Lanes of a warp that carry the same key are linked to each other first (__match_any_sync); the lowest lane of each
// group then either claims the key's slot and publishes the group's chain, or -- the key exists already -- parks the
// chain in the CTA chain cache.
template <int RPT>
__device__ __forceinline__ void sink_build(const PipelineParams& P, const BuildParams& B, const TileCtx& c, Smem* sm) {
  const uint8_t* pact = P.mask_slot == NO_SLOT ? nullptr : c.arena + eff(c, P.mask_slot);
  const int lane = threadIdx.x & 31;
  ChainCacheEntry* cache = reinterpret_cast<ChainCacheEntry*>(c.arena + B.smem_off);
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    const bool live = r < c.nrows && (pact == nullptr || pact[r]);
    KeyRegs key; bool has_null = false; uint64_t h = 0;
    const long long row = B.row_base + c.row0 + r;
    if (live) { h = pack_key<MAX_KEYS>(B.keys, B.n_keys, 0, c, r, key, &has_null); B.next[row] = -1; }
    const bool ins = live && !has_null;                         // NULL keys never match (NullEqualsNothing)
    const unsigned long long tag = h | 1ull;
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, ins ? tag : (0xFFFFFFFFFFFFFF00ull | (unsigned)lane) & ~1ull);
    const int leader = __ffs(peers) - 1;
    const long long leader_row = __shfl_sync(0xFFFFFFFFu, row, leader);
    // members of a group: the leader and the peers whose key really equals the leader's (equal hash is not enough)
    const bool follower = ins && lane != leader;
    const bool same = follower && build_row_has_key(B.keys, B.key_cols, B.key_stride, B.n_keys, (int64_t)leader_row, key);
    const bool member = ins && (lane == leader || same);
    const unsigned cm = __ballot_sync(0xFFFFFFFFu, member) & peers;
    long long last_row = row;
    if (member) {
      const unsigned above = cm & ~((2u << lane) - 1);          // members in higher lanes: link in lane order
      const int nxt = above ? __ffs(above) - 1 : -1;
      const long long next_row = __shfl_sync(cm, row, nxt >= 0 ? nxt : lane);
      if (nxt >= 0) B.next[row] = next_row;
      last_row = __shfl_sync(cm, row, 31 - __clz(cm));
    }
    if (member && lane == leader) {
      bool pushed;
      uint8_t* slot = build_find_or_claim(B, key, h, row, last_row, &pushed);
      if (slot && !pushed && !chain_cache_push(B, cache, &sm->cache_count, slot, row, last_row)) chain_push(B, slot, row, last_row);
    } else if (follower && !same) {                             // same hash, different key (64-bit collision)
      bool pushed;
      uint8_t* slot = build_find_or_claim(B, key, h, row, row, &pushed);
      if (slot && !pushed) chain_push(B, slot, row, row);
    }
  }
}

// hash of the partition key columns of row r exactly as oracle/ops.py::hash_partition_ids: h = mix64(h ^ colhash)
__device__ __forceinline__ uint32_t partition_of(const PartitionParams& Q, const TileCtx& c, int r) {
  uint64_t h = 0;
  for (int i = 0; i < Q.n_keys; ++i) {
    const KeyDesc& d = Q.keys[i];
    const uint8_t* p = c.arena + eff(c, d.slot) + r * d.stride;
    uint64_t ch;
    const bool isnull = d.valid_slot != NO_SLOT && c.arena[eff(c, d.valid_slot) + r] == 0;
    if (isnull) ch = 0x6E756C6C6E756C6Cull;
    else if (d.width == 16) {
      ulonglong2 v = *reinterpret_cast<const ulonglong2*>(p);
      if (d.is_view) {
        // length-seeded chain over 8-byte little-endian words of the string bytes
        const uint32_t len = (uint32_t)v.x;
        const uint8_t* s = view_ptr(v, p);
        uint64_t x = len;
        for (uint32_t o = 0; o < len; o += 8) {
          uint64_t w = 0;
          for (uint32_t b = 0; b < 8 && o + b < len; ++b) w |= (uint64_t)s[o + b] << (8 * b);
          x = mix64(x ^ w);
        }
        ch = mix64(x);
      } else ch = mix64(v.x ^ mix64(v.y));
    } else if (d.width == 8) ch = mix64(lds<uint64_t>(p));
    else if (d.width == 4) ch = mix64((uint64_t)(int64_t)lds<int32_t>(p));
    else ch = mix64((uint64_t)*p);
    h = mix64(h ^ ch);
  }
  return (uint32_t)(h % (uint64_t)Q.n_parts);
}

// RepartitionExec Hash: per tile, rows are counted per partition in shared memory (warp-aggregated:
// __match_any_sync elects one lane per distinct partition id in the warp), the CTA reserves one contiguous range per
// non-empty partition with a single global atomic, and every row scatters to base[pid] + its rank.
// pass 0 only accumulates the global histogram.
template <int RPT>
__device__ __forceinline__ void sink_partition(const PipelineParams& P, const PartitionParams& Q, const TileCtx& c) {
  const uint8_t* pact = P.mask_slot == NO_SLOT ? nullptr : c.arena + eff(c, P.mask_slot);
  uint32_t* cnt = reinterpret_cast<uint32_t*>(c.arena + Q.smem_off);
  unsigned long long* base = reinterpret_cast<unsigned long long*>(c.arena + Q.smem_off + (((size_t)Q.n_parts * 4 + 7) & ~(size_t)7));
  const int lane = threadIdx.x & 31;
  for (int p = threadIdx.x; p < Q.n_parts; p += NT) cnt[p] = 0;
  __syncthreads();
  uint32_t pid[RPT], rank[RPT];
  bool live[RPT];
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int r = threadIdx.x + k * NT;
    live[k] = r < c.nrows && (pact == nullptr || pact[r]);
    pid[k] = live[k] ? partition_of(Q, c, r) : 0xFFFFFFFFu - lane;       // idle lanes match nobody
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, pid[k]);
    const int leader = __ffs(peers) - 1;
    uint32_t first = 0;
    if (live[k] && lane == leader) first = atomicAdd(&cnt[pid[k]], (uint32_t)__popc(peers));
    first = __shfl_sync(0xFFFFFFFFu, first, leader);
    rank[k] = first + __popc(peers & ((1u << lane) - 1));
  }
  __syncthreads();
  for (int p = threadIdx.x; p < Q.n_parts; p += NT) {
    const uint32_t n = cnt[p];
    if (n) {
      const unsigned long long at = atomicAdd(Q.part_counts + p, (unsigned long long)n);
      if (Q.pass) base[p] = (unsigned long long)Q.part_offsets[p] + at;
    }
  }
  if (Q.pass == 0) { __syncthreads(); return; }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    if (!live[k]) continue;
    const int r = threadIdx.x + k * NT;
    const unsigned long long pos = base[pid[k]] + rank[k];
    for (int j = 0; j < P.n_out; ++j) {
      const OutputCol& o = P.out[j];
      if (o.width) store_value(o, c, r, (int64_t)pos);
      else o.data[pos] = c.arena[eff(c, o.slot) + r];
      if (o.valid_slot != NO_SLOT) o.valid_bytes[pos] = c.arena[eff(c, o.valid_slot) + r];
    }
  }
}

// ================================================================================================
// the kernel
// ================================================================================================
// KC (kernel class) splits the instantiations by sink family: the aggregation kernels carry the register accumulators
// and the bounded-table protocol, the others the ordered compaction / join / partition sinks -- each compiles to less
// code and keeps its registers for what it runs.
enum : int { KC_AGG = 0, KC_OTHER = 1, KC_AGG_COLD = 2 };   // KC_AGG_COLD: global table only (no dictionary, no register accumulators)
template <int RPT, int MINB, int KC>
__global__ void __launch_bounds__(NT, MINB) pipeline_kernel(const __grid_constant__ KernelArgs K, int n_stages) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  Smem* sm = reinterpret_cast<Smem*>(smem_raw);
  uint8_t* arena = smem_raw + SMEM_HDR;
  const PipelineParams& P0 = K.P[0];
  const int tile_rows = RPT * NT;
  const int64_t n_tiles = (P0.n_rows + tile_rows - 1) / tile_rows;
  const bool dynamic = KC == KC_OTHER && P0.sink == SINK_COMPACT && P0.tile_offsets == nullptr;
  // static order walks positions blockIdx.x, +gridDim.x, ...: tile numbers themselves or entries of an explicit list
  const int64_t n_pos = P0.tile_list ? P0.n_list : n_tiles;
  auto tile_of = [&](int64_t pos) -> int64_t { return P0.tile_list ? (int64_t)P0.tile_list[pos] : pos; };
  // bounded aggregation table (AggParams::group_limit): once the table is nearly full this CTA stops taking tiles
  const bool guarded = KC != KC_OTHER && K.aux[0].agg.deferred != nullptr;
  auto groups_now = [&]() -> unsigned long long { return *reinterpret_cast<volatile unsigned long long*>(K.aux[0].agg.n_groups); };
  auto pairs_over = [&]() -> bool {                       // any pair set of a DISTINCT aggregate past its limit
    for (int d = 0; d < K.aux[0].n_distinct; ++d) {
      const AggParams& D = K.aux[0].distinct[d];
      if (*reinterpret_cast<volatile unsigned long long*>(D.n_groups) > D.group_limit) return true;
    }
    return false;
  };
  auto table_full = [&]() -> int { return groups_now() > K.aux[0].agg.group_limit || pairs_over() ? 1 : 0; };
  auto defer_rest = [&](int64_t from) {                   // uniform across the CTA
    if (from >= n_pos) return;
    const AggParams& A = K.aux[0].agg;
    const int64_t cnt = (n_pos - from + gridDim.x - 1) / gridDim.x;
    __syncthreads();
    if (threadIdx.x == 0) sm->tile_base = atomicAdd(A.n_deferred, (unsigned long long)cnt);
    __syncthreads();
    const unsigned long long base = sm->tile_base;
    for (int64_t j = threadIdx.x; j < cnt; j += NT) A.deferred[base + j] = (uint32_t)tile_of(from + j * gridDim.x);
  };

  if (threadIdx.x == 0) {
    mbar_init(&sm->full[0], 1);
    mbar_init(&sm->full[1], 1);
    fence_barrier_init();
    sm->dict_n = 0; sm->dict_lock = 0;
    sm->tile[0] = dynamic ? (int)atomicAdd(P0.ticket, 1u) : (int)blockIdx.x;
    sm->defer[0] = guarded ? table_full() : 0;
  }
  if (KC == KC_AGG && K.aux[0].agg.hot_groups > 0) {
    const AggParams& A = K.aux[0].agg;
    hot_init(hot_dict(A, arena), A.hot_groups, A.n_accs, [&](int j) { return (int)A.accs[j].op; });
  }
  if (KC == KC_OTHER && P0.sink == SINK_BUILD) {
    unsigned long long* z = reinterpret_cast<unsigned long long*>(arena + K.aux[0].build.smem_off);
    for (int i = threadIdx.x; i < CHAIN_CACHE_ENTRIES * 3; i += NT) z[i] = 0ull;
    if (threadIdx.x == 0) sm->cache_count = 0;
  }
  __syncthreads();

  uint32_t tma_bytes = 0;
  for (int i = 0; i < P0.n_inputs; ++i) tma_bytes += tile_bytes_of(P0.in[i], tile_rows);

  // returns true when the tile was copied cooperatively (generic proxy): the caller then needs a CTA barrier before
  // anybody reads it; TMA tiles are ordered by their mbarrier instead
  auto issue = [&](int64_t tile, int stage) -> bool {      // uniform across the CTA
    const PipelineParams& P = K.P[stage];
    const int64_t row0 = tile * tile_rows;
    const int nrows = (int)min((int64_t)tile_rows, P.n_rows - row0);
    if (P.use_tma && nrows == tile_rows) {
      if (threadIdx.x == 0) {
        fence_proxy_async();
        mbar_expect_tx(&sm->full[stage], tma_bytes);
        for (int i = 0; i < P.n_inputs; ++i) {
          const InputCol& in = P.in[i];
          const uint32_t bytes = tile_bytes_of(in, tile_rows);
          const uint8_t* src = in.data + (in.width ? (int64_t)in.width * row0 : (row0 >> 3));
          tma_load_1d(arena + in.slot, src, bytes, &sm->full[stage]);
        }
      }
      return false;
    }
    load_tile_generic(P, arena, row0, nrows);
    return true;
  };

  RegAcc<REG_ACCS> R;
#pragma unroll
  for (int g = 0; g < REG_GROUPS; ++g)
#pragma unroll
    for (int j = 0; j < REG_ACCS; ++j) R.v[g][j] = 0;
  R.rows = 0;
  // `cur` / `nxt` are tile numbers in ticket mode and positions (see n_pos) in static mode
  int64_t cur = sm->tile[0];
  const int64_t n_end = dynamic ? n_tiles : n_pos;
  uint32_t parity[2] = {0, 0};
  int it = 0;
  bool defer = sm->defer[0] != 0;
  if (defer) { defer_rest(cur); cur = n_end; }
  if (cur < n_end && issue(dynamic ? cur : tile_of(cur), 0)) __syncthreads();
  for (;; ++it) {
    if (cur >= n_end) break;
    const int s = (n_stages == 2) ? (it & 1) : 0;
    const PipelineParams& P = K.P[s];
    const PipelineAux* aux = &K.aux[s];
    int64_t nxt;
    if (dynamic) {       // ticket order (decoupled look-back needs tiles to start in order): published through shared memory
      if (threadIdx.x == 0) sm->tile[(it + 1) & 1] = (int)atomicAdd(P.ticket, 1u);
      __syncthreads();
      nxt = sm->tile[(it + 1) & 1];
    } else {
      nxt = cur + gridDim.x;                                  // static stride: no barrier needed
    }
    // the group count is read at the top of the tile and only looked at before barrier (B): its latency is hidden
    unsigned long long g_now = 0;
    bool p_over = false;
    if (guarded && threadIdx.x == 0) { g_now = groups_now(); p_over = pairs_over(); }
    const bool prefetched = n_stages == 2 && nxt < n_end && !defer;
    if (prefetched) issue(dynamic ? nxt : tile_of(nxt), s ^ 1);   // prefetch while this tile is computed (consumed after barrier B)
    const int64_t cur_tile = dynamic ? cur : tile_of(cur);
    TileCtx c;
    c.arena = arena; c.stage_off = 0; c.row0 = cur_tile * tile_rows;
    c.nrows = (int)min((int64_t)tile_rows, P.n_rows - c.row0);
    if (P.use_tma && c.nrows == tile_rows) { mbar_wait(&sm->full[s], parity[s]); parity[s] ^= 1; }

    vm_exec<RPT>(K.prog[s], P.n_inst, c, P, aux);
    if constexpr (KC == KC_AGG_COLD) {
      sink_agg_cold<RPT>(P, aux->agg, c);
    } else if constexpr (KC == KC_AGG) {
      if (aux->agg.reg_path) sink_agg_reg<RPT>(P, aux->agg, c, sm, R);
      else sink_agg<RPT>(P, aux->agg, c, sm);
    } else {
      switch (P.sink) {
        case SINK_STORE: sink_store<RPT>(P, c); break;
        case SINK_COMPACT: sink_compact<RPT>(P, c, sm, cur_tile); break;
        case SINK_BUILD: sink_build<RPT>(P, aux->build, c, sm); break;
        case SINK_PARTITION: sink_partition<RPT>(P, aux->part, c); break;
        default: break;
      }
    }
    if (guarded && threadIdx.x == 0) sm->defer[(it + 1) & 1] = g_now > K.aux[0].agg.group_limit || p_over ? 1 : 0;
    if (KC == KC_OTHER && P.sink == SINK_BUILD && threadIdx.x == 0) sm->defer[(it + 1) & 1] = sm->cache_count > CHAIN_CACHE_ENTRIES / 2 ? 1 : 0;
    __syncthreads();                                          // (B) stage s and scratch are free again
    if (KC == KC_OTHER && P.sink == SINK_BUILD && sm->defer[(it + 1) & 1]) {      // crowded cache: push everything, start over
      chain_cache_flush(aux->build, reinterpret_cast<ChainCacheEntry*>(arena + aux->build.smem_off), &sm->cache_count);
    }
    if (guarded) {
      const bool was = defer;
      defer = sm->defer[(it + 1) & 1] != 0;
      // a tile that is already on its way (prefetched) is still processed; everything after it is handed back
      if (n_stages == 2 ? (was && !prefetched) : defer) { defer_rest(nxt); break; }
    }
    if (n_stages == 1 && nxt < n_end && issue(dynamic ? nxt : tile_of(nxt), 0)) __syncthreads();
    cur = nxt;
  }
  if (KC == KC_OTHER && P0.sink == SINK_BUILD)
    chain_cache_flush(K.aux[0].build, reinterpret_cast<ChainCacheEntry*>(arena + K.aux[0].build.smem_off), &sm->cache_count);
  if (KC == KC_AGG && K.aux[0].agg.hot_groups > 0) {
    const AggParams& A = K.aux[0].agg;
    const HotDict H = hot_dict(A, arena);
    if (A.reg_path) reg_flush(H, A.n_accs, R);
    hot_flush(H, &sm->dict_n, A.hot_groups, A.n_accs, A.key_words, [&](int j) { return (int)A.accs[j].op; }, [&](int j) { return (int)A.accs[j].word; },
              agg_entry_of(P0, A, H));
  }
}

// ================================================================================================
// helper kernels
// ================================================================================================
// grow: move every READY entry of `old` into the (larger, empty) table of `A`
__global__ void agg_rehash_kernel(AggParams A, const uint8_t* old_table, const uint32_t* old_occ, uint64_t old_groups, uint32_t* err) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < old_groups; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t* src = reinterpret_cast<const uint64_t*>(old_table) + (uint64_t)old_occ[i] * A.entry_words;
    KeyRegs key;
    for (int w = 0; w < A.key_words; ++w) key.w[w] = src[2 + w];
    uint64_t* e = find_or_insert<FROM_A, FROM_A>(A, key, hash_packed_key(A, key), err, agg_init(), agg_eq());
    if (!e) continue;
    e[1] = src[1];
    for (int w = 0; w < A.acc_words; ++w) e[2 + A.key_words + w] = src[2 + A.key_words + w];
  }
}

__global__ void agg_migrate_kernel(AggParams A, AggMigrateMap M, const uint8_t* old_table, const uint32_t* old_occ, uint64_t old_groups, uint32_t* err) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < old_groups; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t* src = reinterpret_cast<const uint64_t*>(old_table) + (uint64_t)old_occ[i] * M.old_entry_words;
    KeyRegs key;
    for (int w = 0; w < MAX_KEY_WORDS; ++w) key.w[w] = 0;
    for (int w = 0; w < M.old_key_words; ++w) key.w[w + M.key_shift] = src[2 + w];
    uint64_t* e = find_or_insert<FROM_A, FROM_A>(A, key, hash_packed_key(A, key), err, agg_init(), agg_eq());
    if (!e) continue;
    uint64_t seen = 0;
    for (int j = 0; j < A.n_accs; ++j) {
      for (int w = 0; w < acc_words_of(A.accs[j].op); ++w) e[2 + A.key_words + A.accs[j].word + w] = src[2 + M.old_key_words + M.acc_src_word[j] + w];
      if (M.seen_src[j] == -1) seen |= 1ull << j;
      else if (M.seen_src[j] >= 0) seen |= ((src[1] >> M.seen_src[j]) & 1ull) << j;
    }
    e[1] = seen;
  }
}

// The variance family's state from a count n and double-double sums S = sum x and Q = sum x^2: mean = S / n and
// m2 = Q - S^2 / n, both formed in double-double and rounded once.  An m2 within the rounding error of those sums of zero
// (n * Q * 2^-100) is 0: equal values give exactly 0, and the negative values cancellation could leave never appear.  NaN,
// from a NaN or infinite value or from a square beyond the Float64 range, stays NaN.  n = 0 gives 0 and 0.
__device__ __forceinline__ void variance_moments(double n, double sh, double sl, double qh, double ql, bool want_m2, double* mean, double* m2) {
  if (n == 0.0) { *mean = 0.0; *m2 = 0.0; return; }
  // S / n
  const double q1 = sh / n;
  double rh = sh, rl = sl;
  { const double p = q1 * n; dd_add(rh, rl, -p, -fma(q1, n, -p)); }
  *mean = q1 + (rh + rl) / n;
  if (!want_m2) return;
  // S^2 / n
  double s2h, s2l;
  { const double p = sh * sh; dd_fast_two_sum(p, fma(sh, sh, -p) + 2.0 * sh * sl, s2h, s2l); }
  const double d1 = s2h / n;
  double eh = s2h, el = s2l;
  { const double p = d1 * n; dd_add(eh, el, -p, -fma(d1, n, -p)); }
  double dh, dl;
  dd_fast_two_sum(d1, (eh + el) / n, dh, dl);
  double mh = qh, ml = ql;
  dd_add(mh, ml, -dh, -dl);
  const double v = mh + ml;
  *m2 = v <= fabs(qh) * n * 0x1p-100 ? 0.0 : v;
}

__global__ void agg_extract_kernel(AggParams A, AggExtractParams X, uint64_t n_groups, uint32_t* err) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_groups; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t* e = reinterpret_cast<const uint64_t*>(A.table) + (uint64_t)A.occ[i] * A.entry_words;
    const unsigned long long pos = i;
    const uint64_t seen = e[1];
    const uint64_t* kw = e + 2;
    const uint64_t* aw = e + 2 + A.key_words;
    for (int cidx = 0; cidx < X.n_cols; ++cidx) {
      const AggOutCol& o = X.cols[cidx];
      uint8_t* dst = o.data + pos * o.width;
      bool valid = true;
      if (o.kind == 0) {
        if (A.has_null_word) valid = !((kw[0] >> o.a) & 1);
        const uint64_t* s = kw + o.key_word;
        if (o.width == 16) {
          reinterpret_cast<uint64_t*>(dst)[0] = s[0];
          reinterpret_cast<uint64_t*>(dst)[1] = o.src_words == 2 ? s[1] : (uint64_t)((int64_t)s[0] >> 63);
        }
        else if (o.width == 8) *reinterpret_cast<uint64_t*>(dst) = s[0];
        else if (o.width == 4) *reinterpret_cast<uint32_t*>(dst) = (uint32_t)s[0];
        else if (o.width == 2) *reinterpret_cast<uint16_t*>(dst) = (uint16_t)s[0];      // Int16 / UInt16 group keys
        else *dst = (uint8_t)s[0];
      } else if (o.kind == 1) {
        const AccDesc& d = A.accs[o.a];
        if (d.track_seen) valid = (seen >> o.a) & 1;
        const uint64_t* s = aw + d.word;
        if (o.width == 16) {
          uint64_t lo = s[0], hi = o.src_words == 2 ? s[1] : (uint64_t)((int64_t)s[0] >> 63);
          reinterpret_cast<uint64_t*>(dst)[0] = valid ? lo : 0; reinterpret_cast<uint64_t*>(dst)[1] = valid ? hi : 0;
        } else if (o.width == 8) *reinterpret_cast<uint64_t*>(dst) = valid ? s[0] : 0;
        else if (o.width == 4) *reinterpret_cast<uint32_t*>(dst) = valid ? (uint32_t)s[0] : 0;
        else if (o.width == 2) *reinterpret_cast<uint16_t*>(dst) = valid ? (uint16_t)s[0] : 0;
        else *dst = valid ? (uint8_t)s[0] : 0;
      } else if (o.kind >= 3) {
        const uint64_t cnt = aw[A.accs[o.b].word];
        double mean, m2;
        const uint64_t* sw = aw + A.accs[o.kind == 3 ? o.a : o.c].word;
        const uint64_t* qw = aw + A.accs[o.a].word;
        variance_moments((double)cnt, __longlong_as_double((long long)sw[0]), __longlong_as_double((long long)sw[1]),
                         __longlong_as_double((long long)qw[0]), __longlong_as_double((long long)qw[1]), o.kind == 4 || o.kind == 5, &mean, &m2);
        double x = o.kind == 3 ? mean : m2;
        if (o.kind == 5) {
          const bool pop = o.var & VAR_POP;
          valid = pop ? cnt >= 1 : cnt >= 2;
          x = valid ? m2 / (double)(pop ? cnt : cnt - 1) : 0.0;
          if (o.var & VAR_SQRT) x = sqrt(x);
        }
        *reinterpret_cast<double*>(dst) = x;
      } else {
        const AccDesc& ds = A.accs[o.a];
        const uint64_t cnt = aw[A.accs[o.b].word];
        valid = cnt != 0 && (!ds.track_seen || ((seen >> o.a) & 1));
        if (o.is_float) {
          double sum = __longlong_as_double((long long)aw[ds.word]);
          *reinterpret_cast<double*>(dst) = valid ? sum / (double)cnt : 0.0;
        } else {
          // DecimalAverager: (sum * 10^(s_out - s_in)) / count, truncating toward zero; a product that leaves i128 is an
          // overflow error ("Arithmetic Overflow in AvgAccumulator")
          i128 sum = acc_words_of(ds.op) == 2 ? (i128)(((u128)aw[ds.word + 1] << 64) | aw[ds.word]) : (i128)(int64_t)aw[ds.word];
          i128 mul = (i128)(((u128)o.scale_mul_hi << 64) | o.scale_mul_lo);
          i128 q = 0;
          if (valid) {
            if (mul > 1) { const i128 lim = (i128)(~(u128)0 >> 1) / mul; if (sum > lim || sum < -lim) atomicOr(err, ERR_OVERFLOW); }
            q = (i128)((u128)sum * (u128)mul) / (i128)cnt;
          }
          reinterpret_cast<uint64_t*>(dst)[0] = (uint64_t)(u128)q; reinterpret_cast<uint64_t*>(dst)[1] = (uint64_t)((u128)q >> 64);
        }
      }
      if (o.nullable && o.valid_bytes) o.valid_bytes[pos] = valid ? 1 : 0;
    }
  }
}

// bytes (one per row) -> Arrow bitmap
__global__ void pack_bytes_kernel(const uint8_t* __restrict__ bytes, uint32_t* __restrict__ bits, int64_t n, unsigned long long* null_count) {
  const int lane = threadIdx.x & 31;
  const int64_t n_round = (n + 31) & ~31ll;
  unsigned long long nulls = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_round; i += (int64_t)gridDim.x * blockDim.x) {
    const bool v = i < n && bytes[i] != 0;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, v);
    if (lane == 0) { bits[i >> 5] = b; }
    if (i < n && !v) ++nulls;
  }
  if (null_count && nulls) atomicAdd(null_count, nulls);
}

// Arrow bitmap -> bytes (used when a nullable / boolean column must be row-addressable, e.g. join payloads)
__global__ void unpack_bits_kernel(const uint8_t* __restrict__ bits, uint8_t* __restrict__ bytes, int64_t n, int64_t bit_offset) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i + bit_offset;
    bytes[i] = (bits[b >> 3] >> (b & 7)) & 1;
  }
}

// Utf8View import: turn (buffer_index, offset) of long views into absolute device pointers.
__global__ void resolve_views_kernel(ulonglong2* views, int64_t n, const uint64_t* __restrict__ buffer_bases) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    ulonglong2 v = views[i];
    if ((uint32_t)v.x > 12) {
      const uint32_t buf = (uint32_t)v.y, off = (uint32_t)(v.y >> 32);
      v.y = buffer_bases[buf] + off;
      views[i] = v;
    }
  }
}
// Utf8 (offsets + bytes) -> resolved views
__global__ void utf8_to_views_kernel(const int32_t* __restrict__ offsets, const uint8_t* __restrict__ bytes, ulonglong2* views, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t o = offsets[i];
    const uint32_t len = (uint32_t)(offsets[i + 1] - o);
    const uint8_t* s = bytes + o;
    ulonglong2 v; v.x = len; v.y = 0;
    if (len <= 12) {
      uint64_t a = 0, b = 0;
      for (uint32_t k = 0; k < len && k < 4; ++k) a |= (uint64_t)s[k] << (8 * k);
      for (uint32_t k = 4; k < len; ++k) b |= (uint64_t)s[k] << (8 * (k - 4));
      v.x |= a << 32; v.y = b;
    } else {
      uint64_t a = 0;
      for (uint32_t k = 0; k < 4; ++k) a |= (uint64_t)s[k] << (8 * k);
      v.x |= a << 32; v.y = reinterpret_cast<uint64_t>(s);
    }
    views[i] = v;
  }
}
// Export: lengths of long strings (0 for inline) -> exclusive scan on host side is avoided by a
// single-block scan for small outputs or the two-pass below for large ones.
__global__ void view_long_lengths_kernel(const ulonglong2* __restrict__ views, int64_t n, uint32_t* __restrict__ lens, int all) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t len = (uint32_t)views[i].x;
    lens[i] = (all || len > 12) ? len : 0;
  }
}
// copy long-string bytes into a compact heap at offs[i] and rewrite views to (buffer 0, offset)
__global__ void views_to_arrow_kernel(ulonglong2* views, int64_t n, const uint64_t* __restrict__ offs, uint8_t* heap) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    ulonglong2 v = views[i];
    const uint32_t len = (uint32_t)v.x;
    if (len > 12) {
      const uint8_t* s = reinterpret_cast<const uint8_t*>(v.y);
      uint8_t* d = heap + offs[i];
      for (uint32_t k = 0; k < len; ++k) d[k] = s[k];
      v.y = (uint64_t)0 | (offs[i] << 32);
      views[i] = v;
    }
  }
}
// views -> Utf8 (offsets int32 + bytes)
__global__ void views_to_utf8_kernel(const ulonglong2* __restrict__ views, int64_t n, const uint64_t* __restrict__ offs, int32_t* out_offsets, uint8_t* heap) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t* vp = reinterpret_cast<const uint8_t*>(views + i);
    ulonglong2 v = views[i];
    const uint32_t len = (uint32_t)v.x;
    const uint8_t* s = len <= 12 ? vp + 4 : reinterpret_cast<const uint8_t*>(v.y);
    uint8_t* d = heap + offs[i];
    for (uint32_t k = 0; k < len; ++k) d[k] = s[k];
    out_offsets[i] = (int32_t)offs[i];
    if (i == n - 1) out_offsets[n] = (int32_t)(offs[i] + len);
  }
}

// exclusive scan of u32 or u64 -> u64 (sums wrap modulo 2^64), single kernel, one CTA walking the array (outputs are small/medium;
// large inputs use chunked partial sums: pass 1 per-block totals, pass 2 applies block offsets)
template <typename T>
__global__ void scan_block_totals_kernel(const T* __restrict__ in, int64_t n, uint64_t* __restrict__ block_totals, int64_t per_block) {
  __shared__ unsigned long long ws[32];
  const int64_t b0 = blockIdx.x * per_block, b1 = min(n, b0 + per_block);
  unsigned long long s = 0;
  for (int64_t i = b0 + threadIdx.x; i < b1; i += blockDim.x) s += in[i];
  for (int d = 16; d; d >>= 1) s += __shfl_down_sync(0xFFFFFFFFu, s, d);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) { unsigned long long t = 0; for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += ws[w]; block_totals[blockIdx.x] = t; }
}
template <typename T>
__global__ void scan_apply_kernel(const T* __restrict__ in, int64_t n, const uint64_t* __restrict__ block_offsets, uint64_t* __restrict__ out, int64_t per_block) {
  // one warp per block-chunk walks sequentially in 32-wide steps (chunks are sized so this is cheap)
  const int64_t b0 = blockIdx.x * per_block, b1 = min(n, b0 + per_block);
  const int lane = threadIdx.x;
  unsigned long long run = block_offsets[blockIdx.x];
  for (int64_t i = b0; i < b1; i += 32) {
    const int64_t idx = i + lane;
    const unsigned long long v = idx < b1 ? in[idx] : 0;
    unsigned long long incl = v;
    for (int d = 1; d < 32; d <<= 1) { unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += t; }
    if (idx < b1) out[idx] = run + incl - v;
    run += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
}

// ================================================================================================
// host-callable launchers (C++ linkage inside libsailgpu)
// ================================================================================================
typedef void (*PipelineFn)(const KernelArgs, int);
// register budget variants: MINB = resident CTAs per SM the compiler must allow (2 -> 128 regs, 3 -> 80, 4 -> 64)
// instantiated variants: dictionary aggregation always runs 2 CTAs/SM (128 registers for the accumulators), the
// global-table aggregation 4 CTAs/SM, the streaming sinks whatever shared memory allows (2..4)
static PipelineFn pick_kernel(int rpt, int minb, int sink, bool cold) {
  if (sink == SINK_AGG && cold) return rpt == 1 ? pipeline_kernel<1, 4, KC_AGG_COLD> : rpt == 2 ? pipeline_kernel<2, 4, KC_AGG_COLD> : pipeline_kernel<4, 2, KC_AGG_COLD>;
  if (sink == SINK_AGG) return rpt == 1 ? pipeline_kernel<1, 2, KC_AGG> : rpt == 2 ? pipeline_kernel<2, 2, KC_AGG> : pipeline_kernel<4, 2, KC_AGG>;
  if (minb >= 4 && rpt != 4) return rpt == 1 ? pipeline_kernel<1, 4, KC_OTHER> : pipeline_kernel<2, 4, KC_OTHER>;
  if (minb >= 3) return rpt == 1 ? pipeline_kernel<1, 3, KC_OTHER> : rpt == 2 ? pipeline_kernel<2, 3, KC_OTHER> : pipeline_kernel<4, 3, KC_OTHER>;
  return rpt == 1 ? pipeline_kernel<1, 2, KC_OTHER> : rpt == 2 ? pipeline_kernel<2, 2, KC_OTHER> : pipeline_kernel<4, 2, KC_OTHER>;
}
cudaError_t launch_pipeline(const KernelArgs& K, int rpt, int n_stages, size_t smem_bytes, int grid, int minb, cudaStream_t stream) {
  PipelineFn k = pick_kernel(rpt, minb, K.P[0].sink, K.aux[0].agg.cold_only != 0);
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
  if (e != cudaSuccess) return e;
  k<<<grid, NT, smem_bytes, stream>>>(K, n_stages);
  return cudaGetLastError();
}

int pipeline_max_ctas_per_sm(int rpt, int minb, size_t smem_bytes, int sink, bool cold) {
  PipelineFn k = pick_kernel(rpt, minb, sink, cold);
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k, NT, smem_bytes) != cudaSuccess) return 0;
  return n;
}

// two-pass filter: rows kept per tile = popcount of the tile's slice of the packed mask (one warp per tile)
__global__ void tile_popcount_kernel(const uint32_t* __restrict__ bits, int64_t n_rows, int tile_rows, int64_t n_tiles, uint32_t* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int words_per_tile = tile_rows >> 5;
  const int64_t n_words = (n_rows + 31) >> 5;
  for (int64_t t = warp; t < n_tiles; t += n_warps) {
    uint32_t c = 0;
    for (int w = lane; w < words_per_tile; w += 32) {
      const int64_t g = t * words_per_tile + w;
      if (g < n_words) {
        uint32_t x = bits[g];
        const int64_t rem = n_rows - (g << 5);
        if (rem < 32) x &= (1u << rem) - 1;        // bits past the last row are not rows
        c += __popc(x);
      }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, d);
    if (lane == 0) counts[t] = c;
  }
}
cudaError_t launch_tile_popcount(const uint32_t* bits, int64_t n_rows, int tile_rows, int64_t n_tiles, uint32_t* counts, cudaStream_t s) {
  if (n_tiles == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>((n_tiles * 32 + 255) / 256, grid_cap(8));
  tile_popcount_kernel<<<grid, 256, 0, s>>>(bits, n_rows, tile_rows, n_tiles, counts);
  return cudaGetLastError();
}

cudaError_t launch_agg_rehash(const AggParams& A, const uint8_t* old_table, const uint32_t* old_occ, uint64_t old_groups, uint32_t* err, cudaStream_t s) {
  if (old_groups == 0) return cudaSuccess;
  int grid = (int)std::min<uint64_t>((old_groups + 255) / 256, grid_cap(8));
  agg_rehash_kernel<<<grid, 256, 0, s>>>(A, old_table, old_occ, old_groups, err);
  return cudaGetLastError();
}
cudaError_t launch_agg_migrate(const AggParams& A_new, const AggMigrateMap& M, const uint8_t* old_table, const uint32_t* old_occ, uint64_t old_groups, uint32_t* err, cudaStream_t s) {
  if (old_groups == 0) return cudaSuccess;
  int grid = (int)std::min<uint64_t>((old_groups + 255) / 256, grid_cap(8));
  agg_migrate_kernel<<<grid, 256, 0, s>>>(A_new, M, old_table, old_occ, old_groups, err);
  return cudaGetLastError();
}
cudaError_t launch_agg_extract(const AggParams& A, const AggExtractParams& X, uint64_t n_groups, uint32_t* err, cudaStream_t s) {
  if (n_groups == 0) return cudaSuccess;
  int grid = (int)std::min<uint64_t>((n_groups + 255) / 256, grid_cap(8));
  agg_extract_kernel<<<grid, 256, 0, s>>>(A, X, n_groups, err);
  return cudaGetLastError();
}
__global__ void u32_to_bytes_kernel(const uint32_t* __restrict__ in, uint8_t* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = in[i] ? 1 : 0;
}
cudaError_t launch_u32_to_bytes(const uint32_t* in, uint8_t* out, int64_t n, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  u32_to_bytes_kernel<<<(int)std::min<int64_t>((n + 255) / 256, grid_cap(8)), 256, 0, s>>>(in, out, n);
  return cudaGetLastError();
}
cudaError_t launch_pack_bytes(const uint8_t* bytes, uint32_t* bits, int64_t n, unsigned long long* null_count, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  pack_bytes_kernel<<<grid, 256, 0, s>>>(bytes, bits, n, null_count);
  return cudaGetLastError();
}
cudaError_t launch_unpack_bits(const uint8_t* bits, uint8_t* bytes, int64_t n, int64_t bit_offset, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  unpack_bits_kernel<<<grid, 256, 0, s>>>(bits, bytes, n, bit_offset);
  return cudaGetLastError();
}
cudaError_t launch_resolve_views(void* views, int64_t n, const uint64_t* bases, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  resolve_views_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<ulonglong2*>(views), n, bases);
  return cudaGetLastError();
}
cudaError_t launch_utf8_to_views(const int32_t* offsets, const uint8_t* bytes, void* views, int64_t n, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  utf8_to_views_kernel<<<grid, 256, 0, s>>>(offsets, bytes, reinterpret_cast<ulonglong2*>(views), n);
  return cudaGetLastError();
}
__global__ void scan_totals_kernel(uint64_t* t, int64_t nb) {
  const int lane = threadIdx.x; unsigned long long run = 0;
  for (int64_t i = 0; i < nb; i += 32) {
    const int64_t idx = i + lane; const unsigned long long v = idx < nb ? t[idx] : 0; unsigned long long incl = v;
    for (int d = 1; d < 32; d <<= 1) { unsigned long long x = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += x; }
    if (idx < nb) t[idx] = run + incl - v;
    run += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
  if (lane == 0) t[nb] = run;     // grand total after the offsets
}
// exclusive scan of u32 lengths (or u64 values, wrapping) into u64 offsets; block_scratch[nblocks] receives the grand total
template <typename T>
static cudaError_t launch_exclusive_scan(const T* in, int64_t n, uint64_t* out, uint64_t* block_scratch /* >= 1025 u64 */, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  const int64_t nblocks = std::min<int64_t>(1024, (n + 4095) / 4096);
  const int64_t per_block = (n + nblocks - 1) / nblocks;
  scan_block_totals_kernel<T><<<(int)nblocks, 256, 0, s>>>(in, n, block_scratch, per_block);
  scan_totals_kernel<<<1, 32, 0, s>>>(block_scratch, nblocks);
  scan_apply_kernel<T><<<(int)nblocks, 32, 0, s>>>(in, n, block_scratch, out, per_block);
  return cudaGetLastError();
}
cudaError_t launch_exclusive_scan_u32(const uint32_t* in, int64_t n, uint64_t* out, uint64_t* block_scratch, cudaStream_t s) {
  return launch_exclusive_scan(in, n, out, block_scratch, s);
}
cudaError_t launch_exclusive_scan_u64(const uint64_t* in, int64_t n, uint64_t* out, uint64_t* block_scratch, cudaStream_t s) {
  return launch_exclusive_scan(in, n, out, block_scratch, s);
}
cudaError_t launch_view_lengths(const void* views, int64_t n, uint32_t* lens, int all, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  view_long_lengths_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const ulonglong2*>(views), n, lens, all);
  return cudaGetLastError();
}
cudaError_t launch_views_to_arrow(void* views, int64_t n, const uint64_t* offs, uint8_t* heap, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  views_to_arrow_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<ulonglong2*>(views), n, offs, heap);
  return cudaGetLastError();
}
cudaError_t launch_views_to_utf8(const void* views, int64_t n, const uint64_t* offs, int32_t* out_offsets, uint8_t* heap, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  int grid = (int)std::min<int64_t>((n + 255) / 256, grid_cap(8));
  views_to_utf8_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const ulonglong2*>(views), n, offs, out_offsets, heap);
  return cudaGetLastError();
}

}  // namespace sg
