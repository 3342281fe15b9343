// jit_rt.cuh -- device runtime of the SPECIALISED pipeline kernels.
//
// pipeline.cu interprets a fused Filter -> Projection -> Aggregate chain (a tile VM over shared-memory slots, sinks
// driven by descriptors).  For inputs that are worth a second of compilation the host generates, per distinct pipeline,
// a struct `G` (jit.cu) and compiles `jit_main<G>` with NVRTC for sm_90a: expressions become straight-line register
// code (no slots, no dispatch), every descriptor a compile-time constant, and the tile loop becomes an mbarrier ring of
// TMA stages without a CTA-wide barrier per tile (warps drift independently; thread 0 re-arms a stage as soon as all
// eight warps have released it).  The kernel argument block (KernelArgs) is the interpreter's: the generated code reads
// only pointers and sizes from it, so the host-side launch path is shared.
//
// Same operator semantics as pipeline.cu (reference: DataFusion FilterExec / ProjectionExec / AggregateExec as driven by
// crates/sail-execution/src/job_runner.rs:64); the two kernels share the group-table layout and can serve one operator.
#pragma once
#include "agg_hot.cuh"

namespace sg {

// G::Key (jit.cu): the packed key words in registers, padded with zeros to HOT_KEY_WORDS in the dictionary tiers
template <int N> using JitKey = KeyWords<N>;

template <int I> struct IC { static constexpr int value = I; __device__ constexpr operator int() const { return I; } };
template <int I, int N, class F> __device__ __forceinline__ void static_for(F&& f) {
  if constexpr (I < N) { f(IC<I>{}); static_for<I + 1, N>(f); }
}

constexpr int JIT_MAX_STAGES = 4;
constexpr int JIT_NWARPS = NT / 32;
struct JitSmem {
  uint64_t full[JIT_MAX_STAGES];       // "tile landed" (TMA transaction barrier, 1 arrival)
  uint64_t empty[JIT_MAX_STAGES];      // "stage released" (one arrival per warp)
  long long tile_no[JIT_MAX_STAGES];   // tile number of the stage (bit 62: partial tile, copied cooperatively); -1 = end
  unsigned long long tile_base;        // COMPACT: exclusive prefix of the tile
  uint32_t warp_sums[33];
  uint32_t dict_n;                     // groups in the CTA dictionary (release/acquire)
  uint32_t dict_lock;
};
constexpr int JIT_HDR = 256;
static_assert(sizeof(JitSmem) <= JIT_HDR, "JitSmem header");     // jit.hpp: JIT_HDR_BYTES
constexpr long long JIT_PARTIAL = 1ll << 62;

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ---- expression helpers (one call per generated statement) --------------------------------------
__device__ __forceinline__ ulonglong2 mkv16(uint64_t lo, uint64_t hi) { ulonglong2 v; v.x = lo; v.y = hi; return v; }
__device__ __forceinline__ i128 jit_mulw(int64_t a, int64_t b) {
  return mk128((unsigned long long)a * (unsigned long long)b, (unsigned long long)__mul64hi((long long)a, (long long)b));
}
__device__ __forceinline__ i128 jit_mul128_64(i128 a, int64_t b) {
  const unsigned long long alo = (unsigned long long)(u128)a, ahi = (unsigned long long)((u128)a >> 64), ub = (unsigned long long)b;
  return mk128(alo * ub, __umul64hi(alo, ub) + ahi * ub - (b < 0 ? alo : 0ull));
}
template <typename T> __device__ __forceinline__ T jit_divround(T a, T d) {
  T q = a / d, rem = a % d;
  T twice = rem < 0 ? -rem * 2 : rem * 2;
  if (twice >= d) q += (a < 0 ? -1 : 1);
  return q;
}
template <typename T, bool REM> __device__ __forceinline__ T jit_div(T a, T b, bool live, uint32_t* err) {
  return checked_div<T>(a, b, REM, live, err);
}
template <typename D, typename S> __device__ __forceinline__ D jit_cvt(S v) {
  // mirrors the interpreter's OP_CVT: integers widen through i128, floats go through int64 towards integers
  constexpr bool sf = sizeof(S) == 8 && (S)0.5 != (S)0, sf32 = sizeof(S) == 4 && (S)0.5 != (S)0;
  constexpr bool df = sizeof(D) == 8 && (D)0.5 != (D)0;
  if constexpr (sf || sf32) {
    const double fv = (double)v;
    if constexpr (df) return fv;
    else if constexpr (sizeof(D) == 16) return (D)(int64_t)fv;
    else if constexpr (sizeof(D) == 1) return (D)(fv != 0.0);
    else return (D)fv;
  } else {
    if constexpr (df) { if constexpr (sizeof(S) == 16) return (double)v; else return (double)(int64_t)v; }
    else if constexpr (sizeof(D) == 1) return (D)(v != 0);
    else return (D)v;
  }
}
__device__ __forceinline__ int32_t jit_date_part(int32_t days, int part) {
  int y, m, d;
  civil_from_days(days, y, m, d);
  return part == 0 ? y : part == 1 ? m : d;
}
// LIKE over a view held in registers: inline strings are matched from a local copy
__device__ __noinline__ bool jit_like(ulonglong2 v, const uint8_t* pat, uint32_t plen, int cls) {
  const uint32_t len = (uint32_t)v.x;
  if (len > 12) return like_match(reinterpret_cast<const uint8_t*>(v.y), len, pat, plen, cls);
  uint8_t tmp[12];
#pragma unroll
  for (int i = 0; i < 4; ++i) tmp[i] = (uint8_t)(v.x >> (32 + 8 * i));
#pragma unroll
  for (int i = 0; i < 8; ++i) tmp[4 + i] = (uint8_t)(v.y >> (8 * i));
  return like_match(tmp, len, pat, plen, cls);
}

// ================================================================================================
// global group table (agg_hot.cuh), constants from G
// ================================================================================================
// G's arguments to the group-table functions: identities of its accumulators, its key comparison
template <class G>
__device__ __forceinline__ auto jit_init() {
  return [](const AggParams&, uint64_t* acc) {
    static_for<0, G::N_ACCS>([&](auto Jc) { constexpr int J = decltype(Jc)::value;
#pragma unroll
      for (int w = 0; w < acc_words_of(G::acc_op(J)); ++w) acc[G::acc_word(J) + w] = acc_identity(G::acc_op(J), w);
    });
  };
}
template <class G>
__device__ __forceinline__ auto jit_eq() {
  return [](const AggParams&, const uint64_t* k, const typename G::Key& key) { return G::keys_equal(k, key); };
}
// entry_of(g): the table entry of dictionary group g (agg_hot.cuh: hot_entry)
template <class G>
__device__ __forceinline__ auto jit_entry_of(const KernelArgs& K, const HotDict& H) {
  return [&K, H](int g) {
    return hot_entry<G::ENTRY_WORDS, G::KEY_WORDS, typename G::Key>(H, g, K.aux[0].agg, K.P[0].error_flag,
                                                                      [](const AggParams&, const typename G::Key& k) { return G::key_hash(k); }, jit_init<G>(), jit_eq<G>());
  };
}

// warp-level pre-aggregation of one accumulator (jit_cold_rows): `prepare` turns a row's value into a partial state (count(*) of
// one row = 1), `merge` folds another lane's partial state in, `jit_acc_global_n` applies a partial state to the table entry
template <class G, int J>
__device__ __forceinline__ void jit_acc_prepare(AccVal& v) {
  constexpr int op = G::acc_op(J);
  if constexpr (op == ACC_COUNT) { v.i = v.valid ? 1 : 0; }
  else if constexpr (op == ACC_SUM_I64 || op == ACC_SUM_I128) { if (!v.valid) v.i = 0; }
  else if constexpr (op == ACC_SUM_F64) { if (!v.valid) v.f = 0.0; }
  else if constexpr (acc_is_dd(op)) { if (!v.valid) { v.f = 0.0; v.i = 0; } }
}
template <class G, int J>
__device__ __forceinline__ void jit_acc_merge(AccVal& a, const AccVal& b) {
  constexpr int op = G::acc_op(J);
  if constexpr (op == ACC_COUNT || op == ACC_SUM_I64 || op == ACC_SUM_I128) { a.i += b.i; a.valid = a.valid || b.valid; }
  else if constexpr (op == ACC_SUM_F64) { a.f += b.f; a.valid = a.valid || b.valid; }
  else if constexpr (op == ACC_MIN_I32 || op == ACC_MIN_I64 || op == ACC_MIN_I128) { if (b.valid && (!a.valid || b.i < a.i)) { a.i = b.i; a.valid = true; } }
  else if constexpr (op == ACC_MAX_I32 || op == ACC_MAX_I64 || op == ACC_MAX_I128) { if (b.valid && (!a.valid || b.i > a.i)) { a.i = b.i; a.valid = true; } }
  else if constexpr (op == ACC_MIN_F64) { if (b.valid && (!a.valid || b.f < a.f)) { a.f = b.f; a.valid = true; } }
  else if constexpr (op == ACC_MAX_F64) { if (b.valid && (!a.valid || b.f > a.f)) { a.f = b.f; a.valid = true; } }
  else if constexpr (acc_is_dd(op)) {
    double h = a.f, l = __longlong_as_double((long long)i128_lo(a.i));
    dd_add(h, l, b.f, __longlong_as_double((long long)i128_lo(b.i)));
    a.f = h; a.i = (i128)(uint64_t)__double_as_longlong(l); a.valid = a.valid || b.valid;
  }
}
template <class G, int J>
__device__ __forceinline__ void jit_acc_global_n(uint64_t* e, const AccVal& v) {
  constexpr int op = G::acc_op(J);
  if constexpr (op == ACC_COUNT) { if (v.valid) acc_apply(op, e + 2 + G::KEY_WORDS + G::acc_word(J), i128_lo(v.i), 0); }
  else acc_global(e, G::KEY_WORDS, op, G::acc_word(J), J, G::acc_seen(J) != 0, v);
}

// rows whose group is not in the dictionary (or every row of the high-cardinality variant): global table
template <class G>
__device__ __forceinline__ void jit_cold_rows(const KernelArgs& K, const typename G::Row (&rows)[G::RPT], const int (&gid)[G::RPT]) {
  const AggParams& A = K.aux[0].agg;
  uint64_t hh[G::RPT];
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) {
    hh[k] = 0;
    if (rows[k].live && gid[k] < 0) {
      typename G::Key kw;
      G::key_words(rows[k], kw);
      hh[k] = G::key_hash(kw);
      const uint64_t idx = hh[k] & A.capacity_mask;
      prefetch_l2(A.state + idx);
      prefetch_l2(reinterpret_cast<const uint64_t*>(A.table) + idx * G::ENTRY_WORDS);
    }
  }
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) {
    const bool cold = rows[k].live && gid[k] < 0;
    if (__any_sync(0xFFFFFFFFu, cold)) {
      typename G::Key kw;
      G::key_words(rows[k], kw);
      uint64_t* e = find_or_insert_warp<G::ENTRY_WORDS, G::KEY_WORDS>(A, kw, hh[k], cold, K.P[0].error_flag, jit_init<G>(), jit_eq<G>());
      // Rows of one group that sit in the same warp (clustered inputs: the 1-7 lineitems of an order are neighbours) are combined
      // in registers first: one set of accumulator atomics per (warp, group) instead of per row.  The atomics are what bounds this
      // path -- every accumulator adds atomics on top of the inserts.
      const bool upd = cold && e != nullptr;
      const unsigned lane = threadIdx.x & 31;
      const unsigned peers = __match_any_sync(0xFFFFFFFFu, upd ? reinterpret_cast<unsigned long long>(e) : (0xFFFFFFFF00000000ull | lane));
      const int leader = __ffs(peers) - 1;
      const bool solo = peers == (1u << lane);
      if (__all_sync(0xFFFFFFFFu, solo)) {
        if (upd) static_for<0, G::N_ACCS>([&](auto Jc) { constexpr int J = decltype(Jc)::value;
          acc_global(e, G::KEY_WORDS, G::acc_op(J), G::acc_word(J), J, G::acc_seen(J) != 0, G::template acc<J>(rows[k]));
        });
      } else {
        static_for<0, G::N_ACCS>([&](auto Jc) { constexpr int J = decltype(Jc)::value;
          AccVal v = G::template acc<J>(rows[k]);
          if (!upd) v.valid = false;
          jit_acc_prepare<G, J>(v);
          for (unsigned rest = peers & ~(1u << leader); rest; rest &= rest - 1) {      // same trip count for every lane of a peer group
            const int src = __ffs(rest) - 1;
            AccVal o;
            o.i = mk128(__shfl_sync(peers, i128_lo(v.i), src), __shfl_sync(peers, i128_hi(v.i), src));
            o.f = __shfl_sync(peers, v.f, src);
            o.valid = __shfl_sync(peers, (int)v.valid, src) != 0;
            if ((int)lane == leader) jit_acc_merge<G, J>(v, o);
          }
          if (upd && (int)lane == leader) jit_acc_global_n<G, J>(e, v);
        });
      }
    }
  }
}

// per-thread register partials of the integer fast path (tier 2)
template <class G> using JitAggRegs = RegAcc<(G::N_ACCS > 0 ? G::N_ACCS : 1)>;

// tier 2: counts / integer / decimal sums, first REG_GROUPS groups in registers
template <class G>
__device__ __forceinline__ void jit_agg_reg_tile(const KernelArgs& K, const typename G::Row (&rows)[G::RPT], JitSmem* sm, uint8_t* scratch, JitAggRegs<G>& R) {
  static_assert(sizeof(typename G::Key) == sizeof(HotKey), "dictionary tiers hold keys of at most HOT_KEY_WORDS words");
  const HotDict H = hot_dict(scratch, G::HOT_G);
  bool live[G::RPT];
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) live[k] = rows[k].live;
  int gid[G::RPT];
  hot_assign<REG_GROUPS>(H, &sm->dict_n, &sm->dict_lock, REG_GROUPS, live, gid, [&](int k, HotKey& kw) { G::key_words(rows[k], kw); });
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) {
    if (rows[k].live && gid[k] >= 0) {
      int64_t val[G::N_ACCS > 0 ? G::N_ACCS : 1] = {};
      static_for<0, G::N_ACCS>([&](auto Jc) { constexpr int J = decltype(Jc)::value;
        constexpr int mode = G::reg_mode(J);
        if constexpr (mode == 0) val[J] = 1;
        else {
          const AccVal a = G::template acc<J>(rows[k]);
          if constexpr (mode == 3) val[J] = (int64_t)a.i;
          else {
            if (fits55(a.i)) val[J] = (int64_t)a.i;
            else {                                               // rare: exact value straight to the table entry
              val[J] = 0;
              uint64_t* e = jit_entry_of<G>(K, H)(gid[k]);
              // (an Int64 sum has one word and is defined mod 2^64: no carry into the next accumulator)
              if (e) acc_apply(G::acc_op(J), e + 2 + G::KEY_WORDS + G::acc_word(J), i128_lo(a.i), i128_hi(a.i));
            }
          }
        }
      });
      reg_add(R, gid[k], val);
    }
  }
  R.rows += G::RPT;
  if (R.rows >= REG_FLUSH) reg_flush(H, G::N_ACCS, R);
  bool anycold = false;
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) anycold |= rows[k].live && gid[k] < 0;
  if (__any_sync(0xFFFFFFFFu, anycold)) jit_cold_rows<G>(K, rows, gid);
}

// tier 1: any accumulator mix, up to HOT_G groups, per-warp accumulators in shared memory (warp-shuffle reductions)
template <class G>
__device__ __forceinline__ void jit_agg_dict_tile(const KernelArgs& K, const typename G::Row (&rows)[G::RPT], JitSmem* sm, uint8_t* scratch) {
  static_assert(sizeof(typename G::Key) == sizeof(HotKey), "dictionary tiers hold keys of at most HOT_KEY_WORDS words");
  const HotDict H = hot_dict(scratch, G::HOT_G);
  bool live[G::RPT];
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) live[k] = rows[k].live;
  int gid[G::RPT];
  hot_assign<G::HOT_G>(H, &sm->dict_n, &sm->dict_lock, G::HOT_G, live, gid, [&](int k, HotKey& kw) { G::key_words(rows[k], kw); });
  const int hot_n = __shfl_sync(0xFFFFFFFFu, (int)lds_acquire_u32(&sm->dict_n), 0);      // every gid of this warp is below it
  bool anyhot = false;
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) anyhot |= rows[k].live && gid[k] >= 0;
  if (__any_sync(0xFFFFFFFFu, anyhot)) {
    static_for<0, G::N_ACCS>([&](auto Jc) { constexpr int J = decltype(Jc)::value;
      AccVal av[G::RPT];
#pragma unroll
      for (int k = 0; k < G::RPT; ++k) {
        av[k].i = 0; av[k].f = 0.0; av[k].valid = false;
        if (rows[k].live && gid[k] >= 0) av[k] = G::template acc<J>(rows[k]);
      }
      hot_fold<G::RPT>(H, G::HOT_G, G::N_ACCS, hot_n, G::KEY_WORDS, G::acc_op(J), G::acc_word(J), J, G::acc_seen(J) != 0, av, gid,
                       jit_entry_of<G>(K, H));
    });
  }
  bool anycold = false;
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) anycold |= rows[k].live && gid[k] < 0;
  if (__any_sync(0xFFFFFFFFu, anycold)) jit_cold_rows<G>(K, rows, gid);
}

// ================================================================================================
// store / compact sinks
// ================================================================================================
template <class G>
__device__ __forceinline__ void jit_store_tile(const KernelArgs& K, const typename G::Row (&rows)[G::RPT], int64_t row0, int nrows) {
  const PipelineParams& P = K.P[0];
  const int lane = threadIdx.x & 31;
  static_for<0, G::N_OUT>([&](auto Jc) { constexpr int J = decltype(Jc)::value;
#pragma unroll
    for (int k = 0; k < G::RPT; ++k) {
      const int r = threadIdx.x + k * NT;
      const bool in = r < nrows;
      if constexpr (G::out_width(J) != 0) { if (in) G::template store<J>(rows[k], P.out[J].data, row0 + r); }
      else {
        const uint32_t bits = __ballot_sync(0xFFFFFFFFu, in && G::template out_bool<J>(rows[k]));
        if (lane == 0 && (r - lane) < nrows) reinterpret_cast<uint32_t*>(P.out[J].data)[(row0 + r) >> 5] = bits;
      }
      if constexpr (G::out_nullable(J) != 0) {
        const uint32_t vb = __ballot_sync(0xFFFFFFFFu, in && G::template out_valid<J>(rows[k]));
        if (lane == 0 && (r - lane) < nrows) reinterpret_cast<uint32_t*>(P.out[J].valid_bytes)[(row0 + r) >> 5] = vb;
      }
    }
  });
}

// order-preserving compaction; all warps of the CTA work on the same tile (two CTA barriers)
template <class G>
__device__ __forceinline__ void jit_compact_tile(const KernelArgs& K, const typename G::Row (&rows)[G::RPT], JitSmem* sm, int64_t tile) {
  const PipelineParams& P = K.P[0];
  bool keep[G::RPT];
#pragma unroll
  for (int k = 0; k < G::RPT; ++k) keep[k] = rows[k].live;
  uint32_t at[G::RPT];
  const unsigned long long base = compact_positions<G::RPT>(P, keep, tile, G::TILE, sm->warp_sums, &sm->tile_base, at);
  static_for<0, G::N_OUT>([&](auto Jc) { constexpr int J = decltype(Jc)::value;
#pragma unroll
    for (int k = 0; k < G::RPT; ++k) {
      if (!keep[k]) continue;
      const int64_t pos = (int64_t)(base + at[k]);
      if constexpr (G::out_width(J) != 0) G::template store<J>(rows[k], P.out[J].data, pos);
      else P.out[J].data[pos] = G::template out_bool<J>(rows[k]) ? 1 : 0;
      if constexpr (G::out_nullable(J) != 0) P.out[J].valid_bytes[pos] = G::template out_valid<J>(rows[k]) ? 1 : 0;
    }
  });
  __syncthreads();      // warp_sums / tile_base are reused by the next tile
}

// ================================================================================================
// the kernel body
// ================================================================================================
template <class G>
__device__ __forceinline__ void jit_main(const KernelArgs& K) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  JitSmem* sm = reinterpret_cast<JitSmem*>(smem_raw);
  uint8_t* scratch = smem_raw + JIT_HDR;
  uint8_t* ring = scratch + G::SCRATCH_BYTES;
  const PipelineParams& P = K.P[0];
  constexpr int S = G::STAGES;
  constexpr int TILE = G::TILE;
  static_assert(S >= 2 && S <= JIT_MAX_STAGES, "stage ring");
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t n_tiles = (P.n_rows + TILE - 1) / TILE;
  const bool dynamic = G::SINK == SINK_COMPACT && P.tile_offsets == nullptr;
  const int64_t n_pos = P.tile_list ? P.n_list : n_tiles;
  const bool guarded = G::SINK == SINK_AGG && K.aux[0].agg.deferred != nullptr;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) { mbar_init(&sm->full[s], 1); mbar_init(&sm->empty[s], JIT_NWARPS); }
    fence_barrier_init();
    sm->dict_n = 0; sm->dict_lock = 0;
  }
  if constexpr (G::SINK == SINK_AGG && G::AGG_TIER > 0) hot_init(hot_dict(scratch, G::HOT_G), G::HOT_G, G::N_ACCS, [](int j) { return G::acc_op(j); });
  __syncthreads();

  // ---- producer (thread 0): hands tiles to stages ------------------------------------------------
  int64_t next_pos = blockIdx.x;
  bool stopped = false;
  auto produce = [&](int j) {
    const int s = j % S;
    long long tn = -1;
    if (!stopped) {
      int64_t pos;
      if (dynamic) pos = (int64_t)atomicAdd(P.ticket, 1u);
      else { pos = next_pos; next_pos += gridDim.x; }
      if (pos >= (dynamic ? n_tiles : n_pos)) stopped = true;
      else if (guarded && *reinterpret_cast<volatile unsigned long long*>(K.aux[0].agg.n_groups) > K.aux[0].agg.group_limit) {
        // bounded table: hand the tiles this CTA still owns back to the host
        const AggParams& A = K.aux[0].agg;
        const int64_t cnt = (n_pos - pos + gridDim.x - 1) / gridDim.x;
        const unsigned long long base = atomicAdd(A.n_deferred, (unsigned long long)cnt);
        for (int64_t q = 0; q < cnt; ++q) {
          const int64_t pp = pos + q * gridDim.x;
          A.deferred[base + q] = P.tile_list ? P.tile_list[pp] : (uint32_t)pp;
        }
        stopped = true;
      } else tn = (dynamic || !P.tile_list) ? pos : (long long)P.tile_list[pos];
    }
    if (tn >= 0) {
      const int64_t row0 = tn * TILE;
      if (P.n_rows - row0 >= TILE) {
        sm->tile_no[s] = tn;
        fence_proxy_async();
        mbar_expect_tx(&sm->full[s], G::TX_BYTES);
        G::issue(ring + (size_t)s * G::STAGE_BYTES, K, row0, &sm->full[s]);
      } else {
        sm->tile_no[s] = tn | JIT_PARTIAL;
        mbar_arrive(&sm->full[s]);
      }
    } else {
      sm->tile_no[s] = -1;
      mbar_arrive(&sm->full[s]);
    }
  };
  if (tid == 0)
    for (int j = 0; j < S - 1; ++j) produce(j);

  JitAggRegs<G> R;
  if constexpr (G::SINK == SINK_AGG && G::AGG_TIER == 2) {
#pragma unroll
    for (int g = 0; g < REG_GROUPS; ++g)
#pragma unroll
      for (int j = 0; j < G::N_ACCS; ++j) R.v[g][j] = 0;
    R.rows = 0;
  }

  for (int it = 0;; ++it) {
    const int s = it % S;
    if (tid == 0) {
      if (it >= 1) mbar_wait(&sm->empty[(it - 1) % S], (uint32_t)(((it - 1) / S) & 1));
      produce(it + S - 1);
    }
    __syncwarp();
    mbar_wait(&sm->full[s], (uint32_t)((it / S) & 1));
    __syncwarp();
    const long long tn = sm->tile_no[s];
    if (tn < 0) break;
    const int64_t tile = tn & ~JIT_PARTIAL;
    const uint8_t* stg = ring + (size_t)s * G::STAGE_BYTES;
    const int64_t row0 = tile * TILE;
    const int nrows = (int)min((int64_t)TILE, P.n_rows - row0);
    if (tn & JIT_PARTIAL) {       // the last tile of the batch: cooperative copy, zero-filled past the end
      __syncthreads();
      G::copy_partial(ring + (size_t)s * G::STAGE_BYTES, K, row0, nrows);
      __syncthreads();
    }
    typename G::Row rows[G::RPT];
#pragma unroll
    for (int k = 0; k < G::RPT; ++k) {
      const int r = tid + k * NT;
      G::eval(stg, r, r < nrows, K, rows[k]);
    }
    if constexpr (G::SINK == SINK_AGG) {
      if constexpr (G::AGG_TIER == 2) jit_agg_reg_tile<G>(K, rows, sm, scratch, R);
      else if constexpr (G::AGG_TIER == 1) jit_agg_dict_tile<G>(K, rows, sm, scratch);
      else {
        int gid[G::RPT];
#pragma unroll
        for (int k = 0; k < G::RPT; ++k) gid[k] = -1;
        jit_cold_rows<G>(K, rows, gid);
      }
    } else if constexpr (G::SINK == SINK_STORE) {
      jit_store_tile<G>(K, rows, row0, nrows);
    } else if constexpr (G::SINK == SINK_COMPACT) {
      jit_compact_tile<G>(K, rows, sm, tile);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm->empty[s]);
  }
  if constexpr (G::SINK == SINK_AGG && G::AGG_TIER > 0) {
    const HotDict H = hot_dict(scratch, G::HOT_G);
    if constexpr (G::AGG_TIER == 2) reg_flush(H, G::N_ACCS, R);
    hot_flush(H, &sm->dict_n, G::HOT_G, G::N_ACCS, G::KEY_WORDS, [](int j) { return G::acc_op(j); }, [](int j) { return G::acc_word(j); },
              jit_entry_of<G>(K, H));
  }
}

// cooperative copy of one column's partial tile (rows >= nrows zero-filled); called by all NT threads
__device__ __forceinline__ void jit_copy_col(uint8_t* dst, const uint8_t* src, uint32_t total, uint32_t valid, bool aligned16) {
  if (aligned16 && (valid & 15u) == 0) {
    for (uint32_t o = threadIdx.x * 16; o < total; o += NT * 16) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (o < valid) v = *reinterpret_cast<const uint4*>(src + o);
      *reinterpret_cast<uint4*>(dst + o) = v;
    }
  } else {
    for (uint32_t o = threadIdx.x; o < total; o += NT) dst[o] = o < valid ? src[o] : 0;
  }
}

}  // namespace sg
