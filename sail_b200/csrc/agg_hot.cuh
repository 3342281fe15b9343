// agg_hot.cuh -- the global group table, the CTA dictionary of hot groups and the accumulator updates of a hash aggregate,
// shared by the interpreted kernel (pipeline.cu) and the specialised kernels (jit_rt.cuh).
//
// Low-cardinality grouping (TPC-H Q1: 4 groups) keeps the first groups a CTA sees in a dictionary in shared memory, laid out
// as hot_scratch_bytes (vm.h) counts it:
//   u32 fp32[8]                  key fingerprints (four arrive in one LDS.128)
//   u64 keys[G][HOT_KEY_WORDS]   keys padded with zeros to HOT_KEY_WORDS words
//   u64 entry[G]                 global table entries (resolved lazily / at flush)
//   u64 wacc[(warp * G + g) * (1 + 2 * n_accs)]   per-warp accumulator blocks: [seen][acc0 lo, hi][acc1 lo, hi]...
// Entries are immutable once published; dict_n is released after the entry is written, so readers need no lock.  Growth
// takes a CTA-wide spin lock, one lane per warp at a time, so no warp waits on a CTA barrier for it.
//
// The functions take the accumulator's operator, word and counts as plain arguments, and small lambdas for what the kernels
// do differently (key packing, hashing and comparison): the interpreter passes its AggParams, the specialised kernel the
// constants of its G, which fold away once inlined.
#pragma once
#include "dev_ops.cuh"

namespace sg {

// A group key in registers, padded with zeros to N words.  Indexed only by constants and passed by value, so that it stays in
// registers -- never a local-memory array.
template <int N> struct KeyWords { uint64_t w[N]; };
using HotKey = KeyWords<HOT_KEY_WORDS>;

__device__ __forceinline__ i128 mk128(uint64_t lo, uint64_t hi) { return (i128)(((u128)hi << 64) | lo); }
__device__ __forceinline__ uint64_t i128_lo(i128 v) { return (uint64_t)(u128)v; }
__device__ __forceinline__ uint64_t i128_hi(i128 v) { return (uint64_t)((u128)v >> 64); }

__device__ __forceinline__ uint32_t lds_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.cta.shared.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
  return v;
}
__device__ __forceinline__ void sts_release_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.cta.shared.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}

// ---- table accumulators ------------------------------------------------------------------------
// an accumulator value in word form: integers as (lo, hi), Float64 in w0, a double-double as (high, low)
__device__ __forceinline__ void acc_val_words(int op, const AccVal& v, uint64_t& w0, uint64_t& w1) {
  const bool isf = op == ACC_SUM_F64 || op == ACC_MIN_F64 || op == ACC_MAX_F64 || acc_is_dd(op);
  w0 = isf ? (uint64_t)__double_as_longlong(v.f) : i128_lo(v.i);
  w1 = acc_is_dd(op) ? i128_lo(v.i) : isf ? 0 : i128_hi(v.i);
}

// atomic update of the table accumulator at `dst` with (w0, w1)
__device__ __forceinline__ void acc_apply(int op, uint64_t* dst, uint64_t w0, uint64_t w1) {
  switch (op) {
    case ACC_SUM_I64: case ACC_COUNT: if (w0) atomicAdd(reinterpret_cast<unsigned long long*>(dst), (unsigned long long)w0); break;
    case ACC_SUM_I128: atomic_add_i128(dst, mk128(w0, w1)); break;
    case ACC_SUM_F64: atomicAdd(reinterpret_cast<double*>(dst), __longlong_as_double((long long)w0)); break;
    case ACC_MIN_I32: case ACC_MIN_I64: atomicMin(reinterpret_cast<long long*>(dst), (long long)w0); break;
    case ACC_MAX_I32: case ACC_MAX_I64: atomicMax(reinterpret_cast<long long*>(dst), (long long)w0); break;
    case ACC_MIN_I128: atomic_minmax_i128(dst, mk128(w0, w1), true); break;
    case ACC_MAX_I128: atomic_minmax_i128(dst, mk128(w0, w1), false); break;
    case ACC_MIN_F64: atomic_minmax_f64(dst, __longlong_as_double((long long)w0), true); break;
    case ACC_MAX_F64: atomic_minmax_f64(dst, __longlong_as_double((long long)w0), false); break;
    case ACC_DD_SUM: case ACC_DD_SQ: atomic_add_dd(dst, __longlong_as_double((long long)w0), __longlong_as_double((long long)w1)); break;
    default: break;
  }
}

__device__ __forceinline__ void acc_mark_seen(uint64_t* e, int j) {
  const unsigned long long bit = 1ull << j;
  if (!(*reinterpret_cast<volatile unsigned long long*>(e + 1) & bit)) atomicOr(reinterpret_cast<unsigned long long*>(e + 1), bit);
}

// one row's value of accumulator j (operator `op`, first word `word`) applied to table entry e
__device__ __forceinline__ void acc_global(uint64_t* e, int key_words, int op, int word, int j, bool seen, const AccVal& v) {
  uint64_t* dst = e + 2 + key_words + word;
  if (op == ACC_COUNT) { if (v.valid) atomicAdd(reinterpret_cast<unsigned long long*>(dst), 1ull); return; }
  if (!v.valid) return;
  uint64_t w0, w1;
  acc_val_words(op, v, w0, w1);
  acc_apply(op, dst, w0, w1);
  if (seen) acc_mark_seen(e, j);
}

// ---- the global group table --------------------------------------------------------------------
constexpr int FROM_A = -1;
// Entry of EW words: [hash][seen bits][KW key words][accumulators], probed linearly from hash & capacity_mask.  EW and KW are
// the specialised kernel's constants; FROM_A reads A.entry_words / A.key_words where they are used, which costs the
// interpreter fewer registers than values held across the probe loop.
// State word: 0 = empty, else (tag30 << 2) | {1 = being written, 2 = ready}.  Carrying the tag in the state lets a thread skip
// a slot that is being written for a different key without waiting on it.
// init(A, acc) writes the accumulator identities of a fresh entry (acc: its first accumulator word); eq(A, k, key) compares the
// key words k of an entry with `key`.  They take A as an argument rather than capturing it: a capture costs the interpreter
// registers.  `claimed` (optional) is set when this call inserted the key: exactly one caller per key sees it.
template <int EW, int KW, class Key, class Init, class Eq>
__device__ __forceinline__ uint64_t* find_or_insert(const AggParams& A, const Key& key, uint64_t h, uint32_t* err, Init init, Eq eq,
                                                    bool* claimed = nullptr) {
  const uint32_t tag = (uint32_t)(h >> 34) << 2;
  uint64_t idx = h & A.capacity_mask;
  uint64_t probes = 0;
  uint32_t spins = 0;
  while (probes <= A.capacity_mask) {
    uint64_t* e = reinterpret_cast<uint64_t*>(A.table) + idx * (EW != FROM_A ? (uint32_t)EW : A.entry_words);
    uint32_t* st = A.state + idx;
    uint32_t s = ld_acquire_u32(st);
    if (s == ST_EMPTY) {
      s = atomicCAS(st, ST_EMPTY, tag | ST_LOCKED);
      if (s == ST_EMPTY) {
        e[0] = h;
        e[1] = 0;                                                   // seen
        if constexpr (KW != FROM_A) {
#pragma unroll
          for (int w = 0; w < KW; ++w) e[2 + w] = key.w[w];
        } else {
          for (int w = 0; w < A.key_words; ++w) e[2 + w] = key.w[w];
        }
        init(A, e + 2 + (KW != FROM_A ? KW : A.key_words));
        st_release_u32(st, tag | ST_READY);                         // release: the entry words above are visible first
        if (claimed) *claimed = true;
        {
          // occupied-slot list: one counter for the whole table, so the increment is aggregated over the lanes
          // that insert in the same step (same-address atomics serialise in one L2 slice)
          const unsigned m = __activemask();
          const unsigned lane = threadIdx.x & 31;
          const int lead = __ffs(m) - 1;
          unsigned long long base = 0;
          if ((int)lane == lead) base = atomicAdd(A.n_groups, (unsigned long long)__popc(m));
          base = __shfl_sync(m, base, lead);
          A.occ[base + __popc(m & ((1u << lane) - 1))] = (uint32_t)idx;
        }
        return e;
      }
    }
    if ((s & ~3u) == tag) {
      if ((s & 3u) == ST_LOCKED) {          // same tag, still being published: look again (bounded)
        if (++spins > (1u << 24)) { atomicOr(err, ERR_TABLE_FULL); return nullptr; }
        __nanosleep(32);
        continue;
      }
      if (e[0] == h && eq(A, e + 2, key)) return e;
    }
    idx = (idx + 1) & A.capacity_mask;
    ++probes;
  }
  atomicOr(err, ERR_TABLE_FULL);
  return nullptr;
}

// Warp-cooperative front end: lanes of one warp that carry the same key hash elect a leader (__match_any_sync); only leaders
// touch the table, followers receive the entry pointer by shuffle.  Removes same-warp contention on a slot that is being
// published.  All 32 lanes must call; lanes without `need` get nullptr.
// `claimed` (optional): this lane's key was inserted by this call -- by the lane itself, never for a follower.
template <int EW, int KW, class Key, class Init, class Eq>
__device__ __forceinline__ uint64_t* find_or_insert_warp(const AggParams& A, const Key& key, uint64_t h, bool need, uint32_t* err,
                                                         Init init, Eq eq, bool* claimed = nullptr) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long probe = need ? h : (0xFFFFFFFF00000000ull | lane);   // idle lanes match nobody useful
  const unsigned peers = __match_any_sync(0xFFFFFFFFu, probe);
  const int leader = __ffs(peers) - 1;
  uint64_t* e = nullptr;
  bool mine = false;
  if (need && (int)lane == leader) e = find_or_insert<EW, KW>(A, key, h, err, init, eq, &mine);
  unsigned long long p = __shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(e), leader);
  uint64_t* got = reinterpret_cast<uint64_t*>(p);
  // same hash but different key (64-bit collision inside one warp): fall back to an own lookup
  if (need && (int)lane != leader && got && !eq(A, got + 2, key)) got = find_or_insert<EW, KW>(A, key, h, err, init, eq, &mine);
  if (claimed) *claimed = mine;
  return need ? got : nullptr;
}

// ---- the dictionary ----------------------------------------------------------------------------
struct HotDict { uint32_t* fp32; uint64_t* keys; uint64_t* entry; uint64_t* wacc; };
__device__ __forceinline__ HotDict hot_dict(uint8_t* scratch, int groups) {
  HotDict h;
  uint8_t* p = scratch;
  h.fp32 = reinterpret_cast<uint32_t*>(p); p += 32;
  h.keys = reinterpret_cast<uint64_t*>(p); p += (size_t)groups * HOT_KEY_WORDS * 8;
  h.entry = reinterpret_cast<uint64_t*>(p); p += (size_t)groups * 8;
  h.wacc = reinterpret_cast<uint64_t*>(p);
  return h;
}
// accumulator block of (warp, group g)
__device__ __forceinline__ uint64_t* hot_block(const HotDict& H, int warp, int g, int groups, int n_accs) {
  return H.wacc + (size_t)(warp * groups + g) * (1 + 2 * n_accs);
}

__device__ __forceinline__ uint32_t hot_fp(const HotKey& kw) {
  uint32_t fp = fold32(kw.w[0]);
  fp = __funnelshift_l(fp, fp, 7) ^ fold32(kw.w[1]);
  fp = __funnelshift_l(fp, fp, 7) ^ fold32(kw.w[2]);
  fp = __funnelshift_l(fp, fp, 7) ^ fold32(kw.w[3]);
  return fp;
}
__device__ __forceinline__ bool hot_verify(const HotDict& H, int g, const HotKey& kw) {
  const ulonglong2* hk = reinterpret_cast<const ulonglong2*>(H.keys + g * HOT_KEY_WORDS);
  const ulonglong2 a = hk[0], b = hk[1];
  return ((a.x ^ kw.w[0]) | (a.y ^ kw.w[1]) | (b.x ^ kw.w[2]) | (b.y ^ kw.w[3])) == 0ull;
}
// group id of the key among the first n (<= CAP) entries, or -1
template <int CAP>
__device__ __forceinline__ int hot_lookup(const HotDict& H, int n, const HotKey& kw, uint32_t fp) {
  const uint4 f0 = *reinterpret_cast<const uint4*>(H.fp32);
  if (n > 0 && f0.x == fp && hot_verify(H, 0, kw)) return 0;
  if (n > 1 && f0.y == fp && hot_verify(H, 1, kw)) return 1;
  if (n > 2 && f0.z == fp && hot_verify(H, 2, kw)) return 2;
  if (n > 3 && f0.w == fp && hot_verify(H, 3, kw)) return 3;
  if constexpr (CAP > 4) {
    const uint4 f1 = *reinterpret_cast<const uint4*>(H.fp32 + 4);
    if (n > 4 && f1.x == fp && hot_verify(H, 4, kw)) return 4;
    if (n > 5 && f1.y == fp && hot_verify(H, 5, kw)) return 5;
    if (n > 6 && f1.z == fp && hot_verify(H, 6, kw)) return 6;
    if (n > 7 && f1.w == fp && hot_verify(H, 7, kw)) return 7;
  }
  return -1;
}
// warp-collective: lanes with `want` find their key in the dictionary or append it while it holds fewer than `cap` (<= CAP)
// entries; returns the group id or -1 (dictionary full).  Out of line (it runs while the dictionary grows), so H and the key
// are passed by value: a reference would keep them in local memory in the caller, stored on every tile.
template <int CAP>
__device__ __noinline__ int hot_dict_add(const HotDict H, uint32_t* dict_n, uint32_t* dict_lock, int cap, bool want, const HotKey kw, uint32_t fp) {
  const int lane = threadIdx.x & 31;
  int g = -1;
  bool gave_up = false;
  for (;;) {
    const bool need = want && g < 0 && !gave_up;
    const unsigned pend = __ballot_sync(0xFFFFFFFFu, need);
    if (!pend) break;
    const int leader = __ffs(pend) - 1;
    if (lane == leader) {
      while (atomicCAS(dict_lock, 0u, 1u) != 0u) __nanosleep(20);
      const int n = (int)lds_acquire_u32(dict_n);
      g = hot_lookup<CAP>(H, n, kw, fp);
      if (g < 0) {
        if (n < cap) {
#pragma unroll
          for (int w = 0; w < HOT_KEY_WORDS; ++w) H.keys[n * HOT_KEY_WORDS + w] = kw.w[w];
          H.fp32[n] = fp;
          H.entry[n] = 0;
          sts_release_u32(dict_n, (uint32_t)(n + 1));
          g = n;
        } else gave_up = true;
      }
      __threadfence_block();
      atomicExch(dict_lock, 0u);
    }
    __syncwarp();
    if (need && lane != leader) {
      const int n = (int)lds_acquire_u32(dict_n);
      g = hot_lookup<CAP>(H, n, kw, fp);
      if (g < 0 && n >= cap) gave_up = true;
    }
  }
  return g;
}

// Warp-collective: gid[k] of every live row k is its group in the dictionary -- appended while the dictionary holds fewer than
// cap (<= CAP) groups -- or -1.  pack(k, kw) packs row k's key.
template <int CAP, int RPT, class Pack>
__device__ __forceinline__ void hot_assign(const HotDict& H, uint32_t* dict_n, uint32_t* dict_lock, int cap, const bool (&live)[RPT],
                                           int (&gid)[RPT], Pack pack) {
  uint32_t fpv[RPT];
  bool miss = false;
  // The lanes of a warp arrive one by one and other warps grow the dictionary meanwhile: lanes that read different sizes
  // would split around the warp collectives below and hang the warp.  Lane 0's reading is broadcast, so that those
  // collectives are executed by all lanes or by none.
  const int n0 = __shfl_sync(0xFFFFFFFFu, (int)lds_acquire_u32(dict_n), 0);
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    gid[k] = -1; fpv[k] = 0;
    if (live[k]) {
      HotKey kw;
      pack(k, kw);
      fpv[k] = hot_fp(kw);
      gid[k] = hot_lookup<CAP>(H, n0, kw, fpv[k]);
      miss |= gid[k] < 0;
    }
  }
  if (n0 < cap && __any_sync(0xFFFFFFFFu, miss)) {
#pragma unroll
    for (int k = 0; k < RPT; ++k) {
      const bool want = live[k] && gid[k] < 0;
      if (__any_sync(0xFFFFFFFFu, want)) {
        HotKey kw;
        pack(k, kw);
        const int g = hot_dict_add<CAP>(H, dict_n, dict_lock, cap, want, kw, fpv[k]);
        if (want) gid[k] = g;
      }
    }
  }
}

// The table entry of dictionary group g, inserted from the dictionary's copy of the key (hashed with hash(A, key)) on first use.
// Other warps store the same pointer meanwhile (a benign race), hence the volatile load.
template <int EW, int KW, class Key, class Hash, class Init, class Eq>
__device__ __noinline__ uint64_t* hot_entry(const HotDict H, int g, const AggParams& A, uint32_t* err, Hash hash, Init init, Eq eq) {
  uint64_t* e = reinterpret_cast<uint64_t*>(*reinterpret_cast<volatile uint64_t*>(H.entry + g));
  if (e) return e;
  Key key;
#pragma unroll
  for (int w = 0; w < (int)(sizeof(Key) / 8); ++w) key.w[w] = (w < (KW != FROM_A ? KW : A.key_words) && w < HOT_KEY_WORDS) ? H.keys[g * HOT_KEY_WORDS + w] : 0ull;
  e = find_or_insert<EW, KW>(A, key, hash(A, key), err, init, eq);
  H.entry[g] = reinterpret_cast<uint64_t>(e);
  return e;
}

// ---- per-warp accumulator blocks ---------------------------------------------------------------
template <class OpOf>
__device__ __forceinline__ void hot_init(const HotDict& H, int groups, int n_accs, OpOf op_of) {
  for (int i = threadIdx.x; i < (NT / 32) * groups; i += NT) {
    uint64_t* wa = H.wacc + (size_t)i * (1 + 2 * n_accs);
    wa[0] = 0;
    for (int j = 0; j < n_accs; ++j) { wa[1 + 2 * j] = acc_identity(op_of(j), 0); wa[2 + 2 * j] = acc_identity(op_of(j), 1); }
  }
}

// Warp-collective: folds accumulator j (operator `op`, first table word `word`) of this warp's rows that hold a hot group
// (gid >= 0; av: their values) into the warp's accumulator blocks: per group, a thread-local partial, a warp reduction and
// lane 0.  A 128-bit sum that does not fit in 55 bits goes to the table entry exactly (entry_of(g)) instead.
template <int RPT, class EntryOf>
__device__ __forceinline__ void hot_fold(const HotDict& H, int groups, int n_accs, int hot_n, int key_words, int op, int word, int j, bool seen,
                                         const AccVal (&av)[RPT], const int (&gid)[RPT], EntryOf entry_of) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  bool ok[RPT];
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    ok[k] = gid[k] >= 0 && av[k].valid;
    if (op == ACC_SUM_I128 && ok[k] && !fits55(av[k].i)) {   // rare: exact value straight to the table
      uint64_t* e = entry_of(gid[k]);
      if (e) { atomic_add_i128(e + 2 + key_words + word, av[k].i); if (seen) atomicOr(reinterpret_cast<unsigned long long*>(e + 1), 1ull << j); }
      ok[k] = false;
    }
  }
  for (int g = 0; g < hot_n; ++g) {
    uint64_t* wa = hot_block(H, warp, g, groups, n_accs);
    uint64_t* slot = wa + 1 + 2 * j;
    bool any = false;
#pragma unroll
    for (int k = 0; k < RPT; ++k) any |= ok[k] && gid[k] == g;
    if (__ballot_sync(0xFFFFFFFFu, any) == 0) continue;
    if (op == ACC_COUNT) {
      int cnt = 0;
#pragma unroll
      for (int k = 0; k < RPT; ++k) cnt += (ok[k] && gid[k] == g) ? 1 : 0;
      cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
      if (lane == 0) slot[0] += (uint64_t)cnt;
    } else if (op == ACC_SUM_I64 || op == ACC_SUM_I128) {
      int64_t part = 0;
#pragma unroll
      for (int k = 0; k < RPT; ++k) part += (ok[k] && gid[k] == g) ? (int64_t)av[k].i : 0;
      part = warp_sum_i64(part);
      if (lane == 0) {
        if (op == ACC_SUM_I64) slot[0] += (uint64_t)part;
        else { const uint64_t lo = slot[0] + (uint64_t)part; slot[1] += (uint64_t)(part >> 63) + (lo < slot[0] ? 1ull : 0ull); slot[0] = lo; }
      }
    } else if (op == ACC_SUM_F64) {
      double part = 0.0;
#pragma unroll
      for (int k = 0; k < RPT; ++k) part += (ok[k] && gid[k] == g) ? av[k].f : 0.0;
      part = warp_sum_f64(part);
      if (lane == 0) slot[0] = (uint64_t)__double_as_longlong(__longlong_as_double((long long)slot[0]) + part);
    } else {   // min / max (rarely hot) and the double-double sums: per thread, then a shuffle tree, then lane 0
      uint64_t w0 = acc_identity(op, 0), w1 = acc_identity(op, 1);
#pragma unroll
      for (int k = 0; k < RPT; ++k) {
        if (ok[k] && gid[k] == g) {
          uint64_t v0, v1;
          acc_val_words(op, av[k], v0, v1);
          acc_combine_words(op, w0, w1, v0, v1);
        }
      }
#pragma unroll
      for (int dlt = 16; dlt; dlt >>= 1) {
        const uint64_t o0 = __shfl_xor_sync(0xFFFFFFFFu, w0, dlt), o1 = __shfl_xor_sync(0xFFFFFFFFu, w1, dlt);
        acc_combine_words(op, w0, w1, o0, o1);
      }
      if (lane == 0) { uint64_t a0 = slot[0], a1 = slot[1]; acc_combine_words(op, a0, a1, w0, w1); slot[0] = a0; slot[1] = a1; }
    }
    if (seen && lane == 0) wa[0] |= 1ull << j;
  }
}

// ---- register tier: counts and integer sums of the first REG_GROUPS groups in per-thread registers ------------------------
// Values are admitted only below 2^55 in magnitude, and the partials go to warp 0's accumulator blocks every REG_FLUSH rows,
// so they never overflow.
constexpr int REG_FLUSH = 224;    // 224 + RPT values below 2^55 cannot overflow 64 bits
template <int NA> struct RegAcc { int64_t v[REG_GROUPS][NA]; int rows; };

// one row's values into the partials of its group g (0 <= g < REG_GROUPS)
template <int NA>
__device__ __forceinline__ void reg_add(RegAcc<NA>& R, int g, const int64_t (&val)[NA]) {
  static_assert(REG_GROUPS == 4, "one case per register group");
  switch (g) {            // only this row's group is touched (divergent, but 4x fewer adds than predication)
    case 0:
#pragma unroll
      for (int j = 0; j < NA; ++j) R.v[0][j] += val[j];
      break;
    case 1:
#pragma unroll
      for (int j = 0; j < NA; ++j) R.v[1][j] += val[j];
      break;
    case 2:
#pragma unroll
      for (int j = 0; j < NA; ++j) R.v[2][j] += val[j];
      break;
    default:
#pragma unroll
      for (int j = 0; j < NA; ++j) R.v[3][j] += val[j];
  }
}

// Warp-collective (full-mask shuffles): nothing in here may depend on the dictionary size, which other warps change
// asynchronously -- every register group is flushed, groups that do not exist yet hold zeros.  The 32 lanes are summed with
// shuffles first, so only one lane per warp touches the shared accumulators.
template <int NA>
__device__ __forceinline__ void reg_flush(const HotDict& H, int n_accs, RegAcc<NA>& R) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int g = 0; g < REG_GROUPS; ++g) {
    uint64_t* wa = H.wacc + (size_t)g * (1 + 2 * n_accs);
#pragma unroll
    for (int j = 0; j < NA; ++j) {
      if (j < n_accs) {
        // |partial| < 2^63 per lane and the warp total may exceed 64 bits: reduce as 128-bit (lo, carry-aware hi)
        const int64_t part = R.v[g][j];
        unsigned long long lo = (unsigned long long)part;
        long long hi = part >> 63;
#pragma unroll
        for (int d = 16; d; d >>= 1) {
          const unsigned long long olo = __shfl_xor_sync(0xFFFFFFFFu, lo, d);
          const long long ohi = __shfl_xor_sync(0xFFFFFFFFu, hi, d);
          const unsigned long long s = lo + olo;
          hi += ohi + (s < lo ? 1 : 0);
          lo = s;
        }
        if (lane == 0 && (lo | (unsigned long long)hi)) {
          unsigned long long* dst = reinterpret_cast<unsigned long long*>(wa + 1 + 2 * j);
          const unsigned long long old = atomicAdd(dst, lo);
          const unsigned long long carry = (old + lo) < old ? 1ull : 0ull;
          const unsigned long long h2 = (unsigned long long)hi + carry;
          if (h2) atomicAdd(dst + 1, h2);
        }
        R.v[g][j] = 0;
      }
    }
  }
  R.rows = 0;
}

// ---- end of kernel: every warp's blocks of every hot group into the global table ------------------------------------------
// Called by the whole CTA; entry_of(g) resolves (inserting if need be) the table entry of group g.
template <class OpOf, class WordOf, class EntryOf>
__device__ __forceinline__ void hot_flush(const HotDict& H, const uint32_t* dict_n, int groups, int n_accs, int key_words,
                                          OpOf op_of, WordOf word_of, EntryOf entry_of) {
  __syncthreads();
  const int n = (int)lds_acquire_u32(dict_n);
  for (int g = threadIdx.x; g < n; g += NT) entry_of(g);
  __syncthreads();
  const int per = n_accs + 1;   // accumulators + the seen word
  for (int p = threadIdx.x; p < n * per; p += NT) {
    const int g = p / per, j = p % per;
    uint64_t* e = reinterpret_cast<uint64_t*>(H.entry[g]);
    if (!e) continue;
    if (j == n_accs) {
      uint64_t seen = 0;
      for (int w = 0; w < NT / 32; ++w) seen |= hot_block(H, w, g, groups, n_accs)[0];
      if (seen) atomicOr(reinterpret_cast<unsigned long long*>(e + 1), (unsigned long long)seen);
      continue;
    }
    const int op = op_of(j);
    uint64_t w0 = acc_identity(op, 0), w1 = acc_identity(op, 1);
    for (int w = 0; w < NT / 32; ++w) {
      const uint64_t* slot = hot_block(H, w, g, groups, n_accs) + 1 + 2 * j;
      acc_combine_words(op, w0, w1, slot[0], slot[1]);
    }
    acc_apply(op, e + 2 + key_words + word_of(j), w0, w1);
  }
}

}  // namespace sg
