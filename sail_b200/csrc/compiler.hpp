// compiler.hpp -- lowers a chain of FilterExec / ProjectionExec / AggregateExec specs into one
// tile-VM program + sink description (vm.h).  Expressions of later stages are inlined over the
// original input columns, so common sub-expressions across operator boundaries are computed once
// (DataFusion materialises `__common_expr_1`, test_tpch.plan.yaml:15; here it stays in shared
// memory).
#pragma once
#include <map>
#include <set>

#include "device.hpp"
#include "expr.hpp"
#include "vm.h"

namespace sg {

struct Val {
  int kind = K_I64;
  int slot = -1;          // slot id (not an offset); -1 => immediate
  int stride = 0;
  int vslot = -1;         // validity B slot id; -1 => never null
  bool is_imm = false;
  uint64_t i0 = 0, i1 = 0;
};

struct SlotInfo {
  uint32_t bytes_per_row;   // 0 => bit-packed (tile_rows / 8 bytes)
  bool is_input;
  uint32_t offset = 0;
};

struct InputReg { int col; bool validity; int slot; uint16_t width; };

struct StageSpec {
  enum Kind { Filter, Projection, Aggregate } kind;
  ExprPtr predicate;                       // Filter
  std::vector<int> projection; bool has_projection = false;
  std::vector<ExprPtr> exprs; std::vector<std::string> names;     // Projection
  // Aggregate
  std::string mode;
  std::vector<ExprPtr> group_exprs; std::vector<std::string> group_names;
  // distinct: count / sum / avg(DISTINCT arg) of a single-mode aggregate (the flag of min / max is dropped while parsing)
  struct Agg { std::string fn, name; ExprPtr arg; DataType input_type; bool has_arg = false; bool distinct = false; };
  std::vector<Agg> aggs;
};

// what one aggregate output column is made of
// kind: 0 group key a (first word b), 1 accumulator a, 2 avg (sum a / count b); the variance family over a count b, a
// double-double sum and sum of squares: 3 the mean (sum a), 4 m2 (sum of squares a, sum c), 5 var / stddev (as 4; var: VAR_*)
struct AggOutSpec { int kind; int a, b; DataType type; bool nullable; DataType in_type; int c = 0; int var = 0; };

// The pipeline before slot ids were rewritten to arena offsets: input of the kernel specialiser (jit.cu), which turns
// slots into registers and needs to know who reads what.
struct JitInfo {
  bool valid = false;
  std::vector<VmInst> prog;          // operands are slot ids
  std::vector<SlotInfo> slots;
  std::vector<InputReg> inputs;      // slot = slot id
  Val mask;                          // slot < 0 && !is_imm: no filter
  std::vector<OutputCol> outs;       // slot / valid_slot are ids
  std::vector<int> out_kinds;        // VmKind of every output value
  AggParams agg{};                   // keys / accs carry slot ids
  bool small_acc[MAX_ACCS] = {};
  std::vector<KeyDesc> keys;
};
struct JitKernel;

struct CompiledPipeline {
  JitInfo jit;
  std::shared_ptr<JitKernel> jit_kernel;   // specialised kernel, once compiled (jit.cu)
  bool jit_failed = false;                 // generation / compilation was refused: stay on the interpreter
  bool jit_checked = false;                // coverage and kernel cache were looked at
  std::vector<VmInst> prog;          // slot ids already rewritten to arena offsets
  std::vector<SlotInfo> slots;
  std::vector<InputReg> inputs;
  int sink = SINK_STORE;
  uint32_t mask_slot = NO_SLOT;
  std::vector<OutputCol> outs;       // STORE / COMPACT / PARTITION (data pointers filled at launch)
  std::vector<DataType> out_types;
  AggParams agg{};                   // SINK_AGG (table pointers filled at launch)
  std::vector<AggOutSpec> agg_outs;
  std::vector<AggParams> distinct;   // SINK_AGG: the pair set of every DISTINCT argument (OP_DISTINCT_FIRST aux = index; tables filled at launch)
  std::map<std::string, int> acc_ident;   // SINK_AGG: "what is accumulated" (function | argument expression) -> accumulator index; the same
                                     // identities exist under every validity signature, which is how a table is carried over when a
                                     // later batch brings validity buffers an earlier one did not have (engine.cu: migrate_layout)
  std::vector<KeyDesc> keys;         // SINK_BUILD / SINK_PARTITION key slots
  std::vector<std::string> literals; // device-resident byte strings (LIKE patterns, long string literals)
  std::vector<std::pair<int, int>> literal_fixups;   // (instruction index, literal index) -> imm1 pointer
  // geometry (chosen by finalize)
  int rpt = 2, n_stages = 2;
  uint32_t temps_bytes = 0, stage_bytes = 0, hot_bytes = 0, arena_bytes = 0;
  size_t smem_bytes = 0;
  bool cold_variant = false;         // SINK_AGG compiled for high cardinality (set before finalize)
  int n_probes = 0;
  uint32_t extra_scratch = 0;        // sink scratch bytes requested by the operator (partition counters)
  uint32_t scratch_off = 0;          // its arena offset (set by finalize)
};

class PipelineCompiler {
 public:
  PipelineCompiler(const Schema& in, const std::vector<bool>& has_validity) : in_(in), has_validity_(has_validity) {
    for (size_t i = 0; i < in.size(); ++i) {
      auto e = std::make_shared<Expr>();
      e->kind = Expr::Col; e->col = (int)i; e->type = in[i].type; e->nullable = has_validity[i];
      bindings_.push_back(e);
    }
  }

  // bindings = expressions (over the ORIGINAL input columns) of the current stage's schema
  std::vector<ExprPtr>& bindings() { return bindings_; }

  ExprPtr substitute(const ExprPtr& e) const {
    if (e->kind == Expr::Col) return bindings_.at((size_t)e->col);
    if (e->kind == Expr::Lit) return e;
    auto c = std::make_shared<Expr>(*e);
    bool nullable = false;
    for (auto& a : c->args) { a = substitute(a); nullable |= a->nullable; }
    // nullability may shrink when the actual batch carries no validity buffers
    if (e->kind != Expr::IsNull && e->kind != Expr::IsNotNull && !(e->kind == Expr::Case && !e->has_else)) c->nullable = nullable;
    return c;
  }

  void add_filter(const ExprPtr& pred_over_stage) {
    Val p = compile(substitute(pred_over_stage));
    Val t = truthy(p);
    mask_ = mask_.slot < 0 && !mask_.is_imm ? t : b_and(mask_, t);
    has_filter_ = true;
  }
  void set_projection(const std::vector<int>& proj) {
    std::vector<ExprPtr> nb;
    for (int i : proj) nb.push_back(bindings_.at((size_t)i));
    bindings_ = nb;
  }
  void set_exprs(const std::vector<ExprPtr>& exprs_over_stage) {
    std::vector<ExprPtr> nb;
    for (auto& e : exprs_over_stage) nb.push_back(substitute(e));
    bindings_ = nb;
  }

  // ---- sinks ------------------------------------------------------------------------------------
  void finish_store_or_compact(CompiledPipeline& out) {
    out.sink = has_filter_ ? SINK_COMPACT : SINK_STORE;
    emit_outputs(out);
  }
  // first pass of the two-pass filter: the only output is the filter mask itself, as a non-null Bool column
  void finish_mask_store(CompiledPipeline& out) {
    DataType bt; bt.id = TypeId::Bool;
    ExprPtr ph = placeholder(90000, bt, false);
    Val mv = ensure_slot(mask_);
    mv.vslot = -1;
    bind_value(ph, mv);
    bindings_ = {ph};
    mask_ = Val{}; has_filter_ = false;
    out.sink = SINK_STORE;
    emit_outputs(out);
  }
  void finish_partition(CompiledPipeline& out, const std::vector<ExprPtr>& key_exprs_over_stage) {
    out.sink = SINK_PARTITION;
    for (auto& e : key_exprs_over_stage) out.keys.push_back(key_desc(compile(substitute(e)), substitute(e)->type));
    emit_outputs(out);
  }
  void finish_build(CompiledPipeline& out, const std::vector<int>& key_cols) {
    out.sink = SINK_BUILD;
    for (int c : key_cols) out.keys.push_back(key_desc(compile(bindings_.at((size_t)c)), bindings_.at((size_t)c)->type));
  }
  void finish_aggregate(CompiledPipeline& out, const StageSpec& st);

  // join probe inside the pipeline: returns (matched B value, row-id I64 value)
  std::pair<Val, Val> add_probe(CompiledPipeline& out, const std::vector<int>& probe_key_cols, ProbeParams& pp) {
    pp.n_keys = (int)probe_key_cols.size();
    for (size_t i = 0; i < probe_key_cols.size(); ++i) {
      const ExprPtr& e = bindings_.at((size_t)probe_key_cols[i]);
      pp.keys[i] = key_desc(compile(e), e->type);
    }
    Val m = temp(K_B), row = temp(K_I64);
    pp.match_slot = (uint32_t)m.slot; pp.rowid_slot = (uint32_t)row.slot;
    VmInst I{}; I.op = OP_PROBE; I.aux = (uint16_t)out.n_probes; I.dst = (uint32_t)m.slot; I.a = (uint32_t)row.slot; I.b = NO_SLOT;
    I.c = mask_.slot >= 0 ? (uint32_t)mask_.slot : NO_SLOT;
    prog_.push_back(I);
    probe_slot_refs_.push_back(out.n_probes);
    out.n_probes++;
    return {m, row};
  }
  // gathered build-side column as a new binding value (device pointer patched at launch through imm1)
  Val add_gather(const Val& row, int kind, int elem_width, int* inst_index) {
    Val d = temp(kind);
    VmInst I{}; I.op = (uint16_t)(OP_GATHER | (kind << 8)); I.aux = (uint16_t)elem_width; I.dst = (uint32_t)d.slot; I.a = (uint32_t)row.slot;
    I.b = NO_SLOT; I.c = NO_SLOT;
    *inst_index = (int)prog_.size();
    prog_.push_back(I);
    return d;
  }
  Val not_val(const Val& v) { return b_not(v); }
  Val and_val(const Val& a, const Val& b) { return b_and(a, b); }
  Val materialize(const Val& v) { return ensure_slot(v); }
  static ExprPtr placeholder(int id, const DataType& t, bool nullable) {
    auto e = std::make_shared<Expr>(); e->kind = Expr::Col; e->col = 100000 + id; e->type = t; e->nullable = nullable; return e;
  }
  void and_mask(const Val& b) { mask_ = (mask_.slot < 0 && !mask_.is_imm) ? b : b_and(mask_, b); has_filter_ = true; }
  void bind_value(const ExprPtr& placeholder, const Val& v) { cse_[placeholder->key()] = v; }

  void finalize(CompiledPipeline& out, Ctx* ctx, int hot_wanted);

  Val compile(const ExprPtr& e);
  Val mask() const { return mask_; }
  bool has_filter() const { return has_filter_; }
  std::vector<VmInst>& prog() { return prog_; }
  std::vector<ProbeParams*> probe_params;   // patched in finalize (slot ids -> offsets)

 private:
  const Schema& in_;
  std::vector<bool> has_validity_;
  std::vector<ExprPtr> bindings_;
  std::vector<VmInst> prog_;
  std::vector<SlotInfo> slots_;
  std::vector<InputReg> inputs_;
  std::map<std::string, Val> cse_;
  std::map<std::pair<int, bool>, int> input_slot_;
  Val mask_;
  bool has_filter_ = false;
  std::vector<std::string> literals_;
  std::vector<std::pair<int, int>> literal_fixups_;
  std::vector<int> probe_slot_refs_;
  size_t state_col_ = 0;               // finish_aggregate, merging: the first input column of the current aggregate's state
  bool small_acc_[MAX_ACCS] = {};      // accumulator input is statically below 2^55 (decimal precision <= 16)
  std::vector<OutputCol> outs_;
  std::vector<DataType> out_types_;
  std::vector<int> out_kinds_;

  static int phys_kind(const DataType& type) {
    const DataType t = type.storage();
    switch (t.id) {
      case TypeId::Bool: return K_B;
      case TypeId::Int8: case TypeId::Int16: case TypeId::Int32: case TypeId::UInt8: case TypeId::UInt16: case TypeId::Date32: return K_I32;
      case TypeId::Int64: case TypeId::UInt32: case TypeId::UInt64: return K_I64;
      case TypeId::Float32: case TypeId::Float64: return K_F64;
      case TypeId::Decimal128: return t.precision <= 18 ? K_I64 : K_I128;
      case TypeId::Utf8: case TypeId::Utf8View: return K_V16;
      default: fail(SAILGPU_ERR_UNSUPPORTED, "type " + t.str() + " is not supported on the GPU path");
    }
  }
  int new_slot(uint32_t bytes_per_row, bool is_input) { slots_.push_back({bytes_per_row, is_input, 0}); return (int)slots_.size() - 1; }
  Val temp(int kind) { Val v; v.kind = kind; v.slot = new_slot((uint32_t)kind_width(kind), false); v.stride = kind_width(kind); return v; }
  static Val imm(int kind, uint64_t i0, uint64_t i1 = 0) { Val v; v.kind = kind; v.is_imm = true; v.i0 = i0; v.i1 = i1; return v; }

  Val input_value(int col);
  Val ensure_slot(const Val& v) {
    if (!v.is_imm) return v;
    Val d = temp(v.kind); d.vslot = v.vslot;
    VmInst I{}; I.op = (uint16_t)(OP_CONST | (v.kind << 8)); I.dst = (uint32_t)d.slot; I.a = I.b = I.c = NO_SLOT; I.imm0 = v.i0; I.imm1 = v.i1;
    prog_.push_back(I);
    return d;
  }
  // generic 2-operand emit (at most one immediate)
  Val emit2(int base, int op_kind, int dst_kind, Val a, Val b, int c_slot = -1, uint16_t aux = 0) {
    if (a.is_imm && b.is_imm) a = ensure_slot(a);
    Val d = temp(dst_kind);
    VmInst I{}; I.op = (uint16_t)(base | (op_kind << 8)); I.aux = aux; I.dst = (uint32_t)d.slot;
    I.a = a.is_imm ? NO_SLOT : (uint32_t)a.slot; I.b = b.is_imm ? NO_SLOT : (uint32_t)b.slot; I.c = c_slot >= 0 ? (uint32_t)c_slot : NO_SLOT;
    I.sa = (uint8_t)a.stride; I.sb = (uint8_t)b.stride;
    if (a.is_imm) { I.flags |= F_IMM_A; I.imm0 = a.i0; I.imm1 = a.i1; }
    if (b.is_imm) { I.flags |= F_IMM_B; I.imm0 = b.i0; I.imm1 = b.i1; }
    prog_.push_back(I);
    return d;
  }
  Val emit1(int base, int op_kind, int dst_kind, Val a, uint16_t aux = 0) {
    a = ensure_slot(a);
    Val d = temp(dst_kind);
    VmInst I{}; I.op = (uint16_t)(base | (op_kind << 8)); I.aux = aux; I.dst = (uint32_t)d.slot; I.a = (uint32_t)a.slot; I.b = I.c = NO_SLOT;
    I.sa = (uint8_t)a.stride;
    prog_.push_back(I);
    return d;
  }
  static uint16_t cvt_src(int kind) { return kind == K_B ? 10 : kind == K_I32 ? 6 : kind == K_I64 ? 7 : kind == K_F64 ? 8 : 9; }
  Val convert(const Val& v, int to_kind) {
    if (v.kind == to_kind) return v;
    if (v.is_imm) {
      Val r = v; r.kind = to_kind;
      if (to_kind == K_F64) { double d = v.kind == K_I128 ? (double)(i128)(((u128)v.i1 << 64) | v.i0) : (double)(int64_t)v.i0; memcpy(&r.i0, &d, 8); r.i1 = 0; }
      else if (v.kind == K_F64) { double d; memcpy(&d, &v.i0, 8); int64_t x = (int64_t)d; r.i0 = (uint64_t)x; r.i1 = (uint64_t)(x >> 63); }
      else if (to_kind == K_I128 && v.kind != K_I128) { r.i1 = (uint64_t)((int64_t)v.i0 >> 63); }
      else if (to_kind == K_I32) { r.i0 = (uint64_t)(int64_t)(int32_t)v.i0; }
      return r;
    }
    Val d = emit1(OP_CVT, to_kind, to_kind, v, cvt_src(v.kind));
    d.vslot = v.vslot;
    return d;
  }
  static Val imm_pow10(int kind, int k) {
    i128 p = pow10_i128(k);
    if (kind == K_F64) { double d = 1.0; for (int i = 0; i < k; ++i) d *= 10.0; uint64_t b; memcpy(&b, &d, 8); return imm(K_F64, b); }
    return imm(kind, (uint64_t)(u128)p, (uint64_t)((u128)p >> 64));
  }
  Val mul_pow10(const Val& v, int k) {   // same kind in/out
    if (k == 0) return v;
    if (v.is_imm) {
      i128 x = (i128)(((u128)v.i1 << 64) | v.i0);
      if (v.kind != K_I128) x = (i128)(int64_t)v.i0;
      x *= pow10_i128(k);
      return imm(v.kind, (uint64_t)(u128)x, (uint64_t)((u128)x >> 64));
    }
    Val d = emit2(OP_MUL, v.kind, v.kind, v, imm_pow10(v.kind, k));
    d.vslot = v.vslot;
    return d;
  }
  int and_valid(int a, int b) {   // slot ids of validity; -1 => always valid
    if (a < 0) return b;
    if (b < 0 || a == b) return a;
    Val x; x.kind = K_B; x.slot = a; x.stride = 1; Val y = x; y.slot = b;
    return emit2(OP_AND, K_B, K_B, x, y).slot;
  }
  Val b_and(const Val& a, const Val& b) { return fold_bool(OP_AND, a, b); }
  Val b_or(const Val& a, const Val& b) { return fold_bool(OP_OR, a, b); }
  Val fold_bool(int base, const Val& a, const Val& b) {
    if (a.is_imm && b.is_imm) return imm(K_B, base == OP_AND ? (a.i0 & b.i0) : (a.i0 | b.i0));
    if (a.is_imm || b.is_imm) {
      const Val& c = a.is_imm ? a : b; const Val& v = a.is_imm ? b : a;
      if (base == OP_AND) return c.i0 ? v : imm(K_B, 0);
      return c.i0 ? imm(K_B, 1) : v;
    }
    if (a.slot == b.slot) return a;
    return emit2(base, K_B, K_B, a, b);
  }
  Val b_not(const Val& a) { if (a.is_imm) return imm(K_B, a.i0 ^ 1); return emit1(OP_NOT, K_B, K_B, a); }
  Val b_andnot(const Val& a, const Val& b) {   // a & !b
    if (b.is_imm) return b.i0 ? imm(K_B, 0) : a;
    if (a.is_imm) return a.i0 ? b_not(b) : imm(K_B, 0);
    return emit2(OP_ANDNOT, K_B, K_B, a, b);
  }
  Val valid_val(const Val& v) { if (v.vslot < 0) return imm(K_B, 1); Val x; x.kind = K_B; x.slot = v.vslot; x.stride = 1; return x; }
  Val value_only(const Val& v) { Val x = v; x.vslot = -1; return x; }
  // predicate is TRUE (not false, not NULL)
  Val truthy(const Val& p) { return p.vslot < 0 ? value_only(p) : b_and(value_only(p), valid_val(p)); }
  int guard_slot(int vslot) {   // rows where a division is actually evaluated: active & operands valid
    Val g = mask_.slot >= 0 || mask_.is_imm ? mask_ : imm(K_B, 1);
    if (vslot >= 0) { Val v; v.kind = K_B; v.slot = vslot; v.stride = 1; g = b_and(g, v); }
    if (g.is_imm) return -1;
    return g.slot;
  }
  KeyDesc key_desc(const Val& v0, const DataType& t) {
    Val v = ensure_slot(v0);
    KeyDesc k{}; k.slot = (uint32_t)v.slot; k.valid_slot = v.vslot >= 0 ? (uint32_t)v.vslot : NO_SLOT;
    k.width = (uint8_t)kind_width(v.kind); k.stride = (uint8_t)v.stride; k.is_view = t.is_string() ? 1 : 0;
    return k;
  }
  void emit_outputs(CompiledPipeline& out) {
    SG_CHECK((int)bindings_.size() <= MAX_OUTPUTS, SAILGPU_ERR_UNSUPPORTED, "more than " + std::to_string(MAX_OUTPUTS) + " output columns");
    for (auto& b : bindings_) {
      Val v = ensure_slot(compile(b));
      OutputCol o{}; o.slot = (uint32_t)v.slot; o.stride = (uint16_t)v.stride; o.valid_slot = v.vslot >= 0 ? (uint32_t)v.vslot : NO_SLOT;
      const DataType& t = b->type;
      SG_CHECK(t.id != TypeId::Float32, SAILGPU_ERR_UNSUPPORTED, "Float32 outputs are not supported yet");
      o.width = (uint16_t)(t.id == TypeId::Bool ? 0 : t.is_string() ? 16 : t.arrow_width());
      outs_.push_back(o);
      out_types_.push_back(t);
      out_kinds_.push_back(v.kind);
    }
    out.outs = outs_; out.out_types = out_types_;
  }
  Val compile_bin(const ExprPtr& e);
  Val compile_cast(const ExprPtr& e);
  // OP_TS_PART / OP_TS_TRUNC over timestamp value `a` of type `t`: unit and zone offset travel in the immediates
  Val ts_op(int base, int dst_kind, int part, const Val& a, const DataType& t);
  Val compile_uncached(const ExprPtr& e);
};

}  // namespace sg
