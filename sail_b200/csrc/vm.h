// vm.h -- structures shared by the host-side pipeline compiler and the device pipeline kernel.
//
// The hot path is ONE kernel shape (pipeline.cu): a persistent CTA walks tiles of TILE rows; the
// referenced input columns of the tile are staged into shared memory by TMA bulk copies
// (cp.async.bulk + mbarrier); a small register-less "tile VM" evaluates the fused
// filter/projection expressions over typed shared-memory slots (thread t owns rows t, t+NT, ...
// of every slot, so no barrier is needed between VM instructions); a sink consumes the tile:
//   SINK_STORE   : ProjectionExec       -- coalesced column stores
//   SINK_COMPACT : FilterExec           -- warp-ballot compaction, order preserving
//                                          (decoupled look-back across tiles)
//   SINK_AGG     : AggregateExec        -- thread-private shared-memory accumulators for hot
//                                          groups, global open-addressing table for the rest
//   SINK_BUILD   : HashJoinExec build   -- key -> row id into a global open-addressing table
//   (probe is a VM instruction: OP_PROBE; hash partition is SINK_PARTITION)
#pragma once
#include <stdint.h>

namespace sg {

constexpr int NT = 256;            // threads per CTA
constexpr int MAX_INPUTS = 20;     // distinct input column buffers staged per tile
constexpr int MAX_OUTPUTS = 24;
constexpr int MAX_KEYS = 6;
constexpr int MAX_KEY_WORDS = 8;   // 64 bytes of packed key
constexpr int MAX_ACCS = 16;
constexpr int MAX_PROBES = 4;
constexpr int MAX_DISTINCT = 4;    // pair sets (distinct arguments) of one aggregate
constexpr int REG_GROUPS = 4;      // hot groups held in registers by the integer fast path
constexpr int REG_ACCS = 6;        // accumulators held in registers per group
constexpr int HOT_KEY_WORDS = 4;   // group keys wider than 32 bytes skip the hot paths (global table only)
constexpr int HOT_MAX_GROUPS = 8;  // groups of the CTA dictionary (agg_hot.cuh): eight fingerprints in two LDS.128
constexpr uint32_t NO_SLOT = 0xFFFFFFFFu;

// shared-memory bytes of a CTA dictionary of `groups` hot groups (agg_hot.cuh): fingerprints, keys, entry pointers and one
// accumulator block per warp and group
__host__ __device__ constexpr uint32_t hot_scratch_bytes(int groups, int n_accs) {
  return groups <= 0 ? 0u : (uint32_t)(32 + groups * (HOT_KEY_WORDS * 8 + 8) + (NT / 32) * groups * (1 + 2 * n_accs) * 8 + 127) & ~127u;
}

enum VmKind : uint8_t { K_B = 0, K_I32 = 1, K_I64 = 2, K_F64 = 3, K_I128 = 4, K_V16 = 5 };
__host__ __device__ inline int kind_width(int k) { return k == K_B ? 1 : k == K_I32 ? 4 : (k == K_I64 || k == K_F64) ? 8 : 16; }

// op = base | kind << 8
enum VmBase : uint16_t {
  OP_NOP = 0,
  OP_UNPACK_BITS,   // dst(B) <- bit-packed tile bits at a
  OP_CONST,         // dst <- imm                                 (kind)
  OP_MOV,           // dst <- a                                   (kind)
  OP_CVT,           // dst(kind) <- convert a(kind2 in `aux`)     int widening / int<->f64 / narrow loads
  OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_REM, OP_NEG,                 // (kind); DIV/REM: c = validity slot or NO_SLOT
  OP_MULW,          // dst(I128) <- a(I64) * b(I64)
  OP_MUL128_64,     // dst(I128) <- a(I128) * b(I64)
  OP_DIVROUND,      // dst <- a / imm rounding half away from zero (decimal rescale down) (kind)
  OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE,                       // dst(B) <- a ? b          (kind of operands)
  OP_AND, OP_OR, OP_NOT, OP_ANDNOT,                               // B slots; ANDNOT: a & !b
  OP_SELECT,        // dst <- c ? a : b                           (kind)
  OP_STR_EQ_LONG,   // dst(B) <- view a == literal (imm0 = len | prefix<<32, imm1 = device ptr)  aux: 1 = negate
  OP_STR_LIKE,      // dst(B) <- view a LIKE pattern; aux = pattern class, imm0 = len, imm1 = device ptr
  OP_DATE_PART,     // dst(I32) <- part(aux: 0 year 1 month 2 day) of Date32 a
  OP_PROBE,         // hash-join probe: aux = probe index (see ProbeParams)
  OP_GATHER,        // dst(kind) <- build column [imm1 ptr] at row id slot a (I64), masked by active; aux = elem width
  OP_SUBSTR,        // dst(V16) <- substr(view a, imm0 = 1-based start character, imm1 = character count or -1): UTF-8 aware
  OP_TS_PART,       // dst(kind: I32, or I64 for TS_SECOND) <- part(aux: TsPart) of timestamp a(I64); imm0 = units per second,
                    //   imm1 = zone offset from UTC in units
  OP_TS_TRUNC,      // dst(I64) <- timestamp a(I64) truncated to part (aux) in the zone; imm0 / imm1 as OP_TS_PART
  OP_MUL_POW10_CHK, // dst(I128) <- a(I128) * imm (a power of ten); ERR_OVERFLOW when a row of c (rows evaluated, or NO_SLOT
                    //   for all) leaves i128: the decimal division rescale that can overflow
  OP_CHAR_LEN,      // dst(I32) <- character_length(view a): UTF-8 characters
  OP_DISTINCT_FIRST,// dst(B) <- the row is active (c: mask slot or NO_SLOT), its DISTINCT argument is valid, and this row claimed
                    //   its (group key, argument) pair in pair set aux (PipelineAux::distinct): true on one row per pair
  OP_COUNT_
};
// OP_TS_PART / OP_TS_TRUNC parts.  TS_SECOND: the part is the microsecond within the minute, the truncation the whole second;
// TS_DAYS (part only): local days since the epoch, the cast to Date32.
enum TsPart : uint16_t { TS_YEAR = 0, TS_QUARTER, TS_MONTH, TS_WEEK, TS_DAY, TS_HOUR, TS_MINUTE, TS_SECOND, TS_DAYS };
enum : uint16_t { F_IMM_A = 1, F_IMM_B = 2 };
// OP_CVT source formats (aux)
enum CvtSrc : uint16_t { SRC_I8 = 0, SRC_I16, SRC_U8, SRC_U16, SRC_U32, SRC_F32, SRC_I32, SRC_I64, SRC_F64, SRC_I128, SRC_B, SRC_U64 };
enum LikeClass : uint16_t { LIKE_EXACT = 0, LIKE_PREFIX = 1, LIKE_SUFFIX = 2, LIKE_CONTAINS = 3, LIKE_GENERIC = 4 };

struct VmInst {
  uint16_t op;       // base | kind << 8
  uint16_t flags;
  uint16_t aux;
  uint8_t sa, sb;    // operand strides in bytes (dst/c use the natural width of their kind)
  uint32_t dst, a, b, c;   // byte offsets into the tile arena
  uint64_t imm0, imm1;     // immediate (low, high)
};
static_assert(sizeof(VmInst) == 40, "VmInst layout");

struct InputCol {
  const uint8_t* data;      // values buffer (or bit-packed bools / validity bits)
  uint32_t slot;            // arena offset the tile lands at
  uint16_t width;           // bytes per row; 0 => bit-packed (tile_rows / 8 bytes per tile)
  uint16_t tma_ok;          // base pointer is 16-byte aligned
};

struct OutputCol {
  uint8_t* data;
  uint8_t* valid_bytes;     // COMPACT: one byte per output row (packed later); STORE: bitmap words
  uint32_t slot;
  uint32_t valid_slot;      // B slot or NO_SLOT
  uint16_t width;           // bytes per row; 0 => boolean column (B slot -> bitmap / bytes)
  uint16_t stride;          // slot stride
};

enum SinkKind : int32_t { SINK_STORE = 0, SINK_COMPACT = 1, SINK_AGG = 2, SINK_BUILD = 3, SINK_PARTITION = 4 };

enum AccOp : uint8_t {
  ACC_SUM_I64 = 0,   // state i64 += value(i64)            (sum of Int*, counts being merged)
  ACC_SUM_I128,      // state i128 += value (i64 or i128 slot; `vkind`)
  ACC_SUM_F64,
  ACC_COUNT,         // state i64 += 1 when value valid (or always when value slot == NO_SLOT)
  ACC_MIN_I64, ACC_MAX_I64, ACC_MIN_I128, ACC_MAX_I128, ACC_MIN_F64, ACC_MAX_F64,
  ACC_MIN_I32, ACC_MAX_I32,
  // variance family: double-double sums (word 0 the high double, word 1 the low one), updated by a 16-byte compare-and-swap
  ACC_DD_SUM,        // state += x                        (merging: += count * mean, formed exactly)
  ACC_DD_SQ          // state += x * x, formed exactly    (merging: += m2 + count * mean^2)
};
__host__ __device__ constexpr bool acc_is_dd(int op) { return op == ACC_DD_SUM || op == ACC_DD_SQ; }
enum : int { VAR_POP = 1, VAR_SQRT = 2 };   // variance outputs: divide by n (else n - 1); take the square root

struct AccDesc {
  uint8_t op;
  uint8_t vkind;           // VmKind of the value slot
  uint8_t stride;          // value slot stride
  uint8_t track_seen;      // set bit `index` of the row's seen word when a value is accumulated
  uint32_t value_slot;     // NO_SLOT for count(*)
  uint32_t valid_slot;     // NO_SLOT => never null
  uint16_t word;           // first 8-byte word of this accumulator inside a global table entry
  uint32_t n_slot;         // ACC_DD_* merging a state row: F64 slots of its count and mean (stride 8); NO_SLOT otherwise
  uint32_t mean_slot;
};

// One 8-byte word of the packed group key: where it is loaded from (static indexing => registers).
struct KeyWord {
  uint32_t slot;
  uint32_t valid_slot;     // NO_SLOT => never null
  uint8_t width;           // bytes to load: 1, 4 or 8
  uint8_t stride;
  uint8_t byte_off;        // 0 or 8: low / high half of a 16-byte element
  uint8_t key_index;
};

struct KeyDesc {
  uint32_t slot;
  uint32_t valid_slot;     // NO_SLOT => never null
  uint8_t width;           // 1,4,8,16
  uint8_t stride;
  uint8_t is_view;         // Utf8View key (inline views compare by value; long strings via pointer)
  uint8_t pad;
};

// Global group table: state[capacity] (u32: 0 empty / 1 being written / 2 ready) kept apart so that a
// worst-case-sized table costs only a 4-byte memset per slot; entries (AoS, written when claimed):
//   [u32 tag | u32 pad][u64 seen][key words][acc words]
struct AggParams {
  int32_t n_keys, n_accs;
  int32_t key_words;       // 8-byte words of packed key (incl. leading null-mask word if has_null_word)
  int32_t acc_words;       // 8-byte words of accumulators
  int32_t has_null_word;
  int32_t hot_groups;      // thread-private slots per CTA (0 disables the hot path)
  KeyDesc keys[MAX_KEYS];
  KeyWord kwords[MAX_KEY_WORDS];
  AccDesc accs[MAX_ACCS];
  int32_t reg_path;        // all accumulators are integer sums/counts: per-thread REGISTER partials for the first
                           // REG_GROUPS hot groups (no shuffles, no shared-memory traffic per row)
  int32_t kw_simple;       // every packed key word is a plain 8-byte load of a never-null column
  // register fast path load plan: mode 0 = constant 1 (count(*)), 1 = i64 slot, 2 = i128 slot, 3 = i64 slot known < 2^55
  struct RegLoad { uint32_t slot; uint16_t stride; uint8_t mode; uint8_t pad; } rload[REG_ACCS];
  uint8_t* table;          // capacity * entry_bytes
  uint32_t* state;         // capacity
  uint32_t* occ;           // slot index of the i-th inserted group (i < *n_groups): extraction walks this, not the table
  uint64_t capacity_mask;  // capacity - 1 (power of two)
  uint32_t entry_words;    // 2 + key_words + acc_words   (8-byte words)
  uint32_t hot_smem_off;   // arena offset of the hot-path scratch
  unsigned long long* n_groups;   // number of occupied entries
  int32_t cold_only;       // high-cardinality variant: no CTA dictionary, every row goes straight to the global table
  // Bounded table: the table is sized for the groups the operator expects, not for its input rows.  A CTA that sees
  // *n_groups above group_limit stops taking tiles and appends the ones it still owned to `deferred`; the host grows the
  // table and re-launches over that list.  group_limit leaves room for every tile that can still be in flight.
  unsigned long long group_limit;
  uint32_t* deferred;             // tile numbers not processed by this launch (null: unguarded launch)
  unsigned long long* n_deferred;
};

// Join hash table (build side): open addressing on a 64-bit key hash.
//   slots[i] = { u64 key_hash_tagged, i64 row } ; unique-key fast path keeps one row per key and
//   flags duplicates in *dup_flag (the host then switches to the chained multi-match path).
struct ProbeParams {
  const uint8_t* table;    // capacity * 16 bytes
  uint64_t capacity_mask;
  int32_t n_keys;
  int32_t join_kind;       // 0 inner (filter + row id), 1 semi (filter), 2 anti (inverse filter), 3 left-outer (row id or -1)
  KeyDesc keys[MAX_KEYS];  // probe-side key slots
  const uint8_t* build_keys[MAX_KEYS];   // build-side key columns (for equality verification)
  uint8_t build_stride[MAX_KEYS];        // their element stride (16 for a <=18-digit decimal compared on its low 8 bytes)
  uint32_t rowid_slot;     // I64 slot receiving the matching build row id
  uint32_t match_slot;     // B slot receiving "matched"
  uint8_t* visited;        // build-side visited bitmap bytes (left/semi/anti emitting build rows) or null
};

struct BuildParams {
  uint8_t* table;
  uint64_t capacity_mask;
  int32_t n_keys;
  KeyDesc keys[MAX_KEYS];
  int64_t row_base;        // global row id of row 0 of this launch
  uint32_t* dup_flag;
  int64_t* next;           // next[row] = next build row with the same key (-1 ends the chain): duplicates cost O(1)
  const uint8_t* key_cols[MAX_KEYS];   // build key columns (to tell "same key" from "same hash" while inserting)
  uint8_t key_stride[MAX_KEYS];
  uint32_t smem_off;       // arena offset of the CTA chain cache (CHAIN_CACHE_BYTES)
};
constexpr uint32_t CHAIN_CACHE_BYTES = 512 * 24;

struct PartitionParams {
  int32_t n_parts;
  int32_t n_keys;
  KeyDesc keys[MAX_KEYS];
  unsigned long long* part_counts;   // [n_parts] histogram (pass 0) / running cursors (pass 1)
  int32_t pass;                      // 0 = histogram only, 1 = scatter using cursors
  const int64_t* part_offsets;       // [n_parts] exclusive offsets into the output columns
  uint32_t pid_slot;
  uint32_t smem_off;                 // arena offset of the per-CTA scratch: u32 cnt[n_parts], u64 base[n_parts]
};

struct PipelineParams {
  int64_t n_rows;
  int32_t tile_rows;       // 256 / 512 / 1024
  int32_t n_inputs;
  int32_t n_inst;
  int32_t sink;
  int32_t use_tma;
  uint32_t arena_bytes;
  uint32_t mask_slot;      // B slot: row is active (passes every fused FilterExec); NO_SLOT => all rows
  const VmInst* prog;
  InputCol in[MAX_INPUTS];
  int32_t n_out;
  OutputCol out[MAX_OUTPUTS];
  // SINK_COMPACT
  unsigned long long* tile_status;   // [n_tiles] decoupled look-back words
  unsigned int* ticket;              // dynamic tile counter
  unsigned long long* out_count;     // total rows kept
  const unsigned long long* tile_offsets;   // COMPACT, two-pass filter: exclusive output offset of every tile (no look-back, static tile order)
  const uint32_t* tile_list;         // static order over an explicit list of tiles (re-launch over deferred tiles) or null
  int64_t n_list;
  uint32_t* error_flag;              // bit 0 divide by zero, bit 1 overflow, bit 2 table full, bit 3 unsupported
  int32_t n_probes;
};

// Large, rarely-touched parameter blocks live in global memory (the kernel parameter space is 4 KB).
struct PipelineAux {
  AggParams agg;
  BuildParams build;
  PartitionParams part;
  ProbeParams probe[MAX_PROBES];
  // DISTINCT aggregates: one pair set per distinct argument -- a group table without accumulators whose key is the group key
  // (always with a null-mask word) followed by the argument.  The descriptors live in device memory (this stage's
  // MAX_DISTINCT entries), so that pipelines without DISTINCT launch with the parameter block they had.
  const AggParams* distinct;
  int32_t n_distinct;
};

// Everything uniform across the grid travels as ONE kernel parameter (constant bank: uniform loads,
// no per-thread cost), pre-resolved on the host for each of the two input stages so the device never
// computes stage-relative offsets.
constexpr int MAX_INST = 64;
struct KernelArgs {
  PipelineParams P[2];
  PipelineAux aux[2];
  VmInst prog[2][MAX_INST];
};

enum : uint32_t { ERR_DIV_ZERO = 1, ERR_OVERFLOW = 2, ERR_TABLE_FULL = 4, ERR_UNSUPPORTED = 8 };

}  // namespace sg
