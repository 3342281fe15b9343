// compiler.cu -- expression -> tile-VM lowering, aggregate sink construction, shared-memory layout.
#include "compiler.hpp"

#include <cstdlib>

#include "kernels.hpp"

namespace sg {

static uint64_t lo64(i128 v) { return (uint64_t)(u128)v; }
static uint64_t hi64(i128 v) { return (uint64_t)((u128)v >> 64); }

Val PipelineCompiler::input_value(int col) {
  const DataType t = in_[(size_t)col].type.storage();
  auto reg = [&](bool validity, uint16_t width) {
    auto key = std::make_pair(col, validity);
    auto it = input_slot_.find(key);
    if (it != input_slot_.end()) return it->second;
    int s = new_slot(width, true);
    input_slot_[key] = s;
    inputs_.push_back({col, validity, s, width});
    SG_CHECK((int)inputs_.size() <= MAX_INPUTS, SAILGPU_ERR_UNSUPPORTED, "pipeline reads more than " + std::to_string(MAX_INPUTS) + " column buffers");
    return s;
  };
  Val v;
  v.kind = phys_kind(t);
  switch (t.id) {
    case TypeId::Bool: {
      int bits = reg(false, 0);
      Val d = temp(K_B);
      VmInst I{}; I.op = OP_UNPACK_BITS; I.dst = (uint32_t)d.slot; I.a = (uint32_t)bits; I.b = I.c = NO_SLOT;
      prog_.push_back(I);
      v = d;
      break;
    }
    case TypeId::Int8: case TypeId::Int16: case TypeId::UInt8: case TypeId::UInt16: case TypeId::UInt32: case TypeId::Float32: {
      const uint16_t w = (uint16_t)t.arrow_width();
      Val raw; raw.slot = reg(false, w); raw.stride = w; raw.kind = v.kind;
      const uint16_t src = t.id == TypeId::Int8 ? SRC_I8 : t.id == TypeId::Int16 ? SRC_I16 : t.id == TypeId::UInt8 ? SRC_U8
                         : t.id == TypeId::UInt16 ? SRC_U16 : t.id == TypeId::UInt32 ? SRC_U32 : SRC_F32;
      v = emit1(OP_CVT, v.kind, v.kind, raw, src);
      break;
    }
    default: {
      const uint16_t w = (uint16_t)(t.is_string() ? 16 : t.arrow_width());
      v.slot = reg(false, w);
      v.stride = w;
    }
  }
  if (has_validity_[(size_t)col]) {
    int bits = reg(true, 0);
    Val d = temp(K_B);
    VmInst I{}; I.op = OP_UNPACK_BITS; I.dst = (uint32_t)d.slot; I.a = (uint32_t)bits; I.b = I.c = NO_SLOT;
    prog_.push_back(I);
    v.vslot = d.slot;
  }
  return v;
}

Val PipelineCompiler::compile(const ExprPtr& e) {
  const std::string k = e->key();
  auto it = cse_.find(k);
  if (it != cse_.end()) return it->second;
  Val v = compile_uncached(e);
  cse_[k] = v;
  return v;
}

Val PipelineCompiler::compile_bin(const ExprPtr& e) {
  const std::string& op = e->op;
  const ExprPtr& le = e->args[0];
  const ExprPtr& re = e->args[1];
  if (is_cmp(op) && le->type.is_string()) {
    // literal longer than 12 bytes: dedicated op with the bytes in device memory
    const ExprPtr* lit = (re->kind == Expr::Lit && !re->lit_null) ? &re : (le->kind == Expr::Lit && !le->lit_null) ? &le : nullptr;
    if (lit && (*lit)->lit_s.size() > 12) {
      Val x = ensure_slot(compile(lit == &re ? le : re));
      Val out = temp(K_B);
      const std::string& s = (*lit)->lit_s;
      uint32_t prefix = 0; memcpy(&prefix, s.data(), 4);
      VmInst I{}; I.op = OP_STR_EQ_LONG; I.aux = op == "!=" ? 1 : 0; I.dst = (uint32_t)out.slot; I.a = (uint32_t)x.slot; I.b = I.c = NO_SLOT;
      I.sa = (uint8_t)x.stride; I.imm0 = (uint64_t)s.size() | ((uint64_t)prefix << 32);
      literal_fixups_.push_back({(int)prog_.size(), (int)literals_.size()});
      literals_.push_back(s);
      prog_.push_back(I);
      out.vslot = x.vslot;
      return out;
    }
  }
  Val l = compile(le), r = compile(re);
  if (op == "and" || op == "or") {
    // Kleene logic: t = definitely true, f = definitely false
    const bool anynull = l.vslot >= 0 || r.vslot >= 0;
    if (!anynull) return fold_bool(op == "and" ? OP_AND : OP_OR, l, r);
    Val lt = truthy(l), rt = truthy(r);
    Val lf = l.vslot >= 0 ? b_andnot(valid_val(l), value_only(l)) : b_not(value_only(l));
    Val rf = r.vslot >= 0 ? b_andnot(valid_val(r), value_only(r)) : b_not(value_only(r));
    Val val, valid;
    if (op == "and") { val = b_and(lt, rt); valid = b_or(val, b_or(lf, rf)); }
    else { val = b_or(lt, rt); valid = b_or(val, b_and(lf, rf)); }
    val = ensure_slot(val);
    if (!valid.is_imm) val.vslot = valid.slot;
    else if (!valid.i0) val.vslot = ensure_slot(valid).slot;
    return val;
  }
  const int vs = and_valid(l.vslot, r.vslot);
  Val d;
  if (is_cmp(op)) {
    const int base = op == "=" ? OP_EQ : op == "!=" ? OP_NE : op == "<" ? OP_LT : op == "<=" ? OP_LE : op == ">" ? OP_GT : OP_GE;
    if (le->type.is_string()) {
      d = emit2(base, K_V16, K_B, l, r);

    } else {
      SG_CHECK(l.kind == r.kind, SAILGPU_ERR_UNSUPPORTED, "comparison operands lowered to different kinds");
      d = emit2(base, l.kind, K_B, l, r);
    }
    d.vslot = vs;
    return d;
  }
  // arithmetic
  const DataType& rt = e->type;
  if (rt.is_decimal()) {
    const DataType &lt = le->type, &rt2 = re->type;
    const int K = phys_kind(rt);
    if (op == "+" || op == "-") {
      Val a = mul_pow10(convert(l, K), rt.scale - lt.scale), b = mul_pow10(convert(r, K), rt.scale - rt2.scale);
      d = emit2(op == "+" ? OP_ADD : OP_SUB, K, K, a, b);
    } else if (op == "*") {
      if (K == K_I64) d = emit2(OP_MUL, K_I64, K_I64, convert(l, K_I64), convert(r, K_I64));
      else if (l.kind == K_I64 && r.kind == K_I64) d = emit2(OP_MULW, K_I128, K_I128, l, r);
      else if (l.kind == K_I128 && r.kind == K_I64) d = emit2(OP_MUL128_64, K_I128, K_I128, ensure_slot(l), r);
      else if (l.kind == K_I64 && r.kind == K_I128) d = emit2(OP_MUL128_64, K_I128, K_I128, ensure_slot(r), l);
      else d = emit2(OP_MUL, K_I128, K_I128, convert(l, K_I128), convert(r, K_I128));
    } else {   // "/" and "%": arrow-arith rescales then divides, truncating
      int lk, rk;
      if (op == "/") { const int mp = rt.scale - lt.scale + rt2.scale; lk = mp > 0 ? mp : 0; rk = mp < 0 ? -mp : 0; }
      else { lk = rt.scale - lt.scale; rk = rt.scale - rt2.scale; }
      const int DK = (lt.precision + lk > 18 || rt2.precision + rk > 18 || K == K_I128) ? K_I128 : K_I64;
      int guard = -2;   // rows evaluated, computed once on first use
      auto rows_evaluated = [&]() { if (guard == -2) guard = guard_slot(vs); return guard; };
      auto rescale = [&](const Val& v, int p, int k) {
        // |v| < 10^p: only where p + k > 38 can the rescale leave i128, and only there is it checked (arrow-rs mul_checked)
        if (p + k <= 38) return mul_pow10(convert(v, DK), k);
        Val d = emit2(OP_MUL_POW10_CHK, K_I128, K_I128, ensure_slot(convert(v, K_I128)), imm_pow10(K_I128, k), rows_evaluated());
        d.vslot = v.vslot;
        return d;
      };
      Val a = rescale(l, lt.precision, lk), b = rescale(r, rt2.precision, rk);
      d = emit2(op == "/" ? OP_DIV : OP_REM, DK, DK, a, b, rows_evaluated());
      d = convert(d, K);
    }
    d.vslot = vs;
    return d;
  }
  SG_CHECK(l.kind == r.kind, SAILGPU_ERR_UNSUPPORTED, "arithmetic operands lowered to different kinds");
  SG_CHECK(le->type.id != TypeId::Float32, SAILGPU_ERR_UNSUPPORTED, "Float32 arithmetic is not supported yet");
  const int K = l.kind;
  if (op == "/" || op == "%") d = emit2(op == "/" ? OP_DIV : OP_REM, K, K, l, r, K == K_F64 ? -1 : guard_slot(vs));
  else d = emit2(op == "+" ? OP_ADD : op == "-" ? OP_SUB : OP_MUL, K, K, l, r);
  d.vslot = vs;
  return d;
}

Val PipelineCompiler::compile_cast(const ExprPtr& e) {
  const ExprPtr& src = e->args[0];
  const DataType &from = src->type, &to = e->type;
  Val v = compile(src);
  const int K = phys_kind(to);
  Val d;
  if (from.is_string() && to.is_string()) return v;
  if (from.is_timestamp() || to.is_timestamp()) {
    // expr.hpp: make_cast admits only these; anything else reaching here is refused rather than relabelled
    if (from.is_timestamp() && to.id == TypeId::Date32) return ts_op(OP_TS_PART, K_I32, TS_DAYS, v, from);
    if (from.is_timestamp() && to.is_timestamp() && to.unit >= from.unit) d = mul_pow10(v, 3 * (to.unit - from.unit));
    else if ((from.is_timestamp() && to.id == TypeId::Int64) || (from.id == TypeId::Int64 && to.is_timestamp())) d = v;   // same value
    else fail(SAILGPU_ERR_UNSUPPORTED, "cast " + from.str() + " -> " + to.str());
    d.vslot = v.vslot;
    return d;
  }
  if (to.is_decimal()) {
    if (from.is_decimal()) {
      if (to.scale >= from.scale) d = mul_pow10(convert(v, K), to.scale - from.scale);
      else {
        Val x = ensure_slot(v);
        Val q = emit2(OP_DIVROUND, x.kind, x.kind, x, imm_pow10(x.kind, from.scale - to.scale));
        d = convert(q, K);
      }
    } else if (from.is_int()) {
      d = mul_pow10(convert(v, K), to.scale);
    } else fail(SAILGPU_ERR_UNSUPPORTED, "cast " + from.str() + " -> " + to.str());
  } else if (to.id == TypeId::Float64) {
    d = convert(v, K_F64);
    if (from.is_decimal() && from.scale > 0) d = emit2(OP_DIV, K_F64, K_F64, d, imm_pow10(K_F64, from.scale));
  } else if (to.is_int() || to.id == TypeId::Date32) {
    if (from.is_decimal()) {
      Val x = v;
      if (from.scale > 0) x = emit2(OP_DIV, v.kind, v.kind, ensure_slot(v), imm_pow10(v.kind, from.scale), -1);
      d = convert(x, K);
    } else d = convert(v, K);
  } else if (to.id == TypeId::Bool && from.id == TypeId::Bool) {
    d = v;
  } else fail(SAILGPU_ERR_UNSUPPORTED, "cast " + from.str() + " -> " + to.str());
  d.vslot = v.vslot;
  return d;
}

Val PipelineCompiler::ts_op(int base, int dst_kind, int part, const Val& a, const DataType& t) {
  const int64_t ups = unit_per_second(t.unit);
  Val d = emit1(base, dst_kind, dst_kind, a, (uint16_t)part);
  prog_.back().imm0 = (uint64_t)ups;
  prog_.back().imm1 = (uint64_t)(zone_offset_seconds(t.tz) * ups);
  d.vslot = a.vslot;
  return d;
}

Val PipelineCompiler::compile_uncached(const ExprPtr& e) {
  switch (e->kind) {
    case Expr::Col: return input_value(e->col);
    case Expr::Lit: {
      const int K = phys_kind(e->type);
      Val v;
      if (e->type.is_string()) {
        SG_CHECK(e->lit_null || e->lit_s.size() <= 12, SAILGPU_ERR_UNSUPPORTED,
                 "string literal longer than 12 bytes outside an equality comparison");
        uint8_t raw[16] = {0};
        const uint32_t len = (uint32_t)e->lit_s.size();
        memcpy(raw, &len, 4);
        memcpy(raw + 4, e->lit_s.data(), len);
        uint64_t a, b; memcpy(&a, raw, 8); memcpy(&b, raw + 8, 8);
        v = imm(K_V16, a, b);
      } else if (K == K_F64) {
        uint64_t b; double d = e->lit_f; memcpy(&b, &d, 8); v = imm(K_F64, b);
      } else {
        v = imm(K, lo64(e->lit_i), hi64(e->lit_i));
      }
      if (e->lit_null) { Val s = ensure_slot(v); s.vslot = ensure_slot(imm(K_B, 0)).slot; return s; }
      return v;
    }
    case Expr::Bin: return compile_bin(e);
    case Expr::Not: { Val a = compile(e->args[0]); Val d = b_not(value_only(a)); d = ensure_slot(d); d.vslot = a.vslot; return d; }
    case Expr::Neg: { Val a = compile(e->args[0]); Val d = emit1(OP_NEG, a.kind, a.kind, a); d.vslot = a.vslot; return d; }
    case Expr::IsNull: { Val a = compile(e->args[0]); return a.vslot < 0 ? imm(K_B, 0) : b_not(valid_val(a)); }
    case Expr::IsNotNull: { Val a = compile(e->args[0]); return a.vslot < 0 ? imm(K_B, 1) : valid_val(a); }
    case Expr::Cast: return compile_cast(e);
    case Expr::Case: {
      const size_t nb = (e->args.size() - (e->has_else ? 1 : 0)) / 2;
      const int K = phys_kind(e->type);
      Val res, resv;
      if (e->has_else) { res = compile(e->args.back()); resv = valid_val(res); res = value_only(res); }
      else { res = imm(K, 0, 0); resv = imm(K_B, 0); }
      for (size_t i = nb; i-- > 0;) {
        Val c = ensure_slot(truthy(compile(e->args[2 * i])));
        Val t = compile(e->args[2 * i + 1]);
        Val tv = valid_val(t);
        Val a = value_only(t), b = res;
        if (a.is_imm && b.is_imm) b = ensure_slot(b);
        res = emit2(OP_SELECT, K, K, a, b, c.slot);
        if (!(tv.is_imm && resv.is_imm && tv.i0 == resv.i0)) {
          Val x = tv, y = resv;
          if (x.is_imm && y.is_imm) y = ensure_slot(y);
          resv = emit2(OP_SELECT, K_B, K_B, x, y, c.slot);
        }
      }
      res = ensure_slot(res);
      if (!(resv.is_imm && resv.i0 == 1)) res.vslot = ensure_slot(resv).slot;
      return res;
    }
    case Expr::Like: {
      Val a = ensure_slot(compile(e->args[0]));
      const std::string& p = e->op;
      // classify: only leading/trailing '%' and no '_' or escapes => fast classes
      std::string body = p;
      bool lead = false, trail = false;
      if (!body.empty() && body.front() == '%') { lead = true; body.erase(0, 1); }
      if (!body.empty() && body.back() == '%' && (body.size() < 2 || body[body.size() - 2] != '\\')) { trail = true; body.pop_back(); }
      int cls;
      if (body.find_first_of("%_\\") != std::string::npos) { cls = LIKE_GENERIC; body = p; }
      else cls = lead && trail ? LIKE_CONTAINS : lead ? LIKE_SUFFIX : trail ? LIKE_PREFIX : LIKE_EXACT;
      Val out = temp(K_B);
      VmInst I{}; I.op = OP_STR_LIKE; I.aux = (uint16_t)(cls | (e->negated ? 0x100 : 0)); I.dst = (uint32_t)out.slot; I.a = (uint32_t)a.slot;
      I.b = I.c = NO_SLOT; I.sa = (uint8_t)a.stride; I.imm0 = body.size();
      literal_fixups_.push_back({(int)prog_.size(), (int)literals_.size()});
      literals_.push_back(body);
      prog_.push_back(I);
      out.vslot = a.vslot;
      return out;
    }
    case Expr::Substr: {
      Val a = ensure_slot(compile(e->args[0]));
      Val out = temp(K_V16);
      VmInst I{}; I.op = (uint16_t)(OP_SUBSTR | (K_V16 << 8)); I.dst = (uint32_t)out.slot; I.a = (uint32_t)a.slot; I.b = I.c = NO_SLOT;
      I.sa = (uint8_t)a.stride; I.imm0 = (uint64_t)e->sub_start; I.imm1 = (uint64_t)e->sub_len;
      prog_.push_back(I);
      out.vslot = a.vslot;
      return out;
    }
    case Expr::CharLength: {
      Val a = ensure_slot(compile(e->args[0]));
      Val out = temp(K_I32);
      VmInst I{}; I.op = (uint16_t)(OP_CHAR_LEN | (K_I32 << 8)); I.dst = (uint32_t)out.slot; I.a = (uint32_t)a.slot; I.b = I.c = NO_SLOT;
      I.sa = (uint8_t)a.stride;
      prog_.push_back(I);
      out.vslot = a.vslot;
      return out;
    }
    case Expr::DateTrunc: {
      const DataType& t = e->args[0]->type;
      return ts_op(OP_TS_TRUNC, K_I64, timestamp_part("date_trunc", e->op), compile(e->args[0]), t);
    }
    case Expr::DatePart: {
      if (e->args[0]->type.is_timestamp()) {
        const int part = timestamp_part("date_part", e->op);
        return ts_op(OP_TS_PART, part == TS_SECOND ? K_I64 : K_I32, part, compile(e->args[0]), e->args[0]->type);
      }
      Val a = compile(e->args[0]);
      Val d = emit1(OP_DATE_PART, K_I32, K_I32, a, (uint16_t)(e->op == "year" ? 0 : e->op == "month" ? 1 : 2));
      d.vslot = a.vslot;
      return d;
    }
  }
  fail(SAILGPU_ERR_INVALID, "bad expression node");
}

// ------------------------------------------------------------------------------------------------
// aggregate sink
// ------------------------------------------------------------------------------------------------
void PipelineCompiler::finish_aggregate(CompiledPipeline& out, const StageSpec& st) {
  out.sink = SINK_AGG;
  AggParams& A = out.agg;
  const bool merging = st.mode == "final" || st.mode == "final_partitioned";
  const bool partial = st.mode == "partial";
  SG_CHECK((int)st.group_exprs.size() <= MAX_KEYS, SAILGPU_ERR_UNSUPPORTED, "more than " + std::to_string(MAX_KEYS) + " group keys");
  A.n_keys = (int)st.group_exprs.size();
  int kw = 0;
  bool any_null_key = false;
  std::vector<int> key_first_word;
  std::vector<DataType> key_types;
  std::vector<ExprPtr> gexprs;
  for (auto& g : st.group_exprs) gexprs.push_back(substitute(g));
  for (size_t i = 0; i < gexprs.size(); ++i) {
    Val v = compile(gexprs[i]);
    A.keys[i] = key_desc(v, gexprs[i]->type);
    any_null_key |= A.keys[i].valid_slot != NO_SLOT;
    key_types.push_back(gexprs[i]->type);
  }
  A.has_null_word = any_null_key ? 1 : 0;
  kw = A.has_null_word;
  for (int i = 0; i < A.n_keys; ++i) { key_first_word.push_back(kw); kw += A.keys[i].width == 16 ? 2 : 1; }
  SG_CHECK(kw <= MAX_KEY_WORDS, SAILGPU_ERR_UNSUPPORTED, "group key wider than " + std::to_string(MAX_KEY_WORDS * 8) + " bytes");
  A.key_words = kw;

  // accumulators, de-duplicated on (op, value slot, validity slot)
  std::map<std::tuple<int, int, int, uint64_t>, int> dedup;
  int words = 0;
  auto add_acc = [&](int op, const Val* value) -> int {
    Val v;
    int vslot = -1, valid = -1, vkind = K_I64, stride = 0;
    if (value) {
      v = ensure_slot(*value);
      vslot = v.slot; valid = v.vslot; vkind = v.kind; stride = v.stride;
    }
    auto key = std::make_tuple(op, vslot, valid, (uint64_t)0);
    auto it = dedup.find(key);
    if (it != dedup.end()) return it->second;
    SG_CHECK(A.n_accs < MAX_ACCS, SAILGPU_ERR_UNSUPPORTED, "more than " + std::to_string(MAX_ACCS) + " distinct accumulators");
    AccDesc d{}; d.op = (uint8_t)op; d.vkind = (uint8_t)vkind; d.stride = (uint8_t)stride;
    d.value_slot = vslot >= 0 ? (uint32_t)vslot : NO_SLOT; d.valid_slot = valid >= 0 ? (uint32_t)valid : NO_SLOT;
    d.n_slot = d.mean_slot = NO_SLOT;
    // a variance accumulator's nulls come from its count
    d.track_seen = (op != ACC_COUNT && !acc_is_dd(op) && (valid >= 0 || A.n_keys == 0)) ? 1 : 0;
    // a 128-bit min / max and a double-double sum are updated by a 16-byte compare-and-swap, which needs a 16-byte aligned
    // address: they start on an even word of their entry (and entries are an even number of words long, below)
    if ((op == ACC_MIN_I128 || op == ACC_MAX_I128 || acc_is_dd(op)) && ((2 + A.key_words + words) & 1)) ++words;
    d.word = (uint16_t)words;
    words += (op == ACC_SUM_I128 || op == ACC_MIN_I128 || op == ACC_MAX_I128 || acc_is_dd(op)) ? 2 : 1;
    A.accs[A.n_accs] = d;
    dedup[key] = A.n_accs;
    return A.n_accs++;
  };
  auto ident = [&](const std::string& what, int j) { out.acc_ident[what] = j; return j; };
  // DISTINCT: one gate per argument (shared by count / sum / avg over it), a B slot that is true on the one row of each
  // (group key, argument) pair that claimed the pair in the argument's pair set.  The gate implies an active row and a valid
  // argument, so it alone is the validity of the gated accumulators: that slot is new, so add_acc never merges a gated
  // accumulator with a plain one over the same argument, and their identities carry "distinct|".
  std::map<std::string, int> gates;
  auto gate_for = [&](const Val& x0, const DataType& t, const std::string& id) -> int {
    auto it = gates.find(id);
    if (it != gates.end()) return it->second;
    SG_CHECK((int)out.distinct.size() < MAX_DISTINCT, SAILGPU_ERR_UNSUPPORTED, "more than " + std::to_string(MAX_DISTINCT) + " DISTINCT arguments in one aggregate");
    const Val x = ensure_slot(x0);
    AggParams D{};
    D.n_keys = A.n_keys + 1;
    SG_CHECK(D.n_keys <= MAX_KEYS, SAILGPU_ERR_UNSUPPORTED, "DISTINCT aggregate: grouping columns plus the argument exceed " + std::to_string(MAX_KEYS) + " columns");
    for (int i = 0; i < A.n_keys; ++i) D.keys[i] = A.keys[i];
    D.keys[A.n_keys] = key_desc(x, t);
    D.has_null_word = 1;            // always: the pair layout does not depend on which batches carry validity buffers
    D.key_words = 1;
    for (int i = 0; i < D.n_keys; ++i) D.key_words += D.keys[i].width == 16 ? 2 : 1;
    SG_CHECK(D.key_words <= MAX_KEY_WORDS, SAILGPU_ERR_UNSUPPORTED, "DISTINCT aggregate: grouping columns plus the argument are wider than " + std::to_string(MAX_KEY_WORDS * 8 - 8) + " bytes");
    D.entry_words = (uint32_t)(2 + D.key_words);
    D.group_limit = ~0ull;
    Val g = temp(K_B);
    VmInst I{}; I.op = OP_DISTINCT_FIRST; I.aux = (uint16_t)out.distinct.size(); I.dst = (uint32_t)g.slot; I.a = I.b = NO_SLOT;
    I.c = (!mask_.is_imm && mask_.slot >= 0) ? (uint32_t)mask_.slot : NO_SLOT;
    prog_.push_back(I);
    out.distinct.push_back(D);
    gates[id] = g.slot;
    return g.slot;
  };
  auto sum_acc = [&](const Val& x, const DataType& t, const std::string& id) -> int {
    if (t.is_decimal()) { const int j = add_acc(ACC_SUM_I128, &x); if (t.precision <= 16 && j < MAX_ACCS) small_acc_[j] = true; return ident("sum|" + id, j); }
    if (t.is_float()) { Val f = convert(x, K_F64); f.vslot = x.vslot; return ident("sum|" + id, add_acc(ACC_SUM_F64, &f)); }
    Val w = convert(x, K_I64); w.vslot = x.vslot;
    return ident("sum|" + id, add_acc(ACC_SUM_I64, &w));
  };
  auto minmax_acc = [&](bool is_min, const Val& x, const DataType& t) -> int {
    SG_CHECK(!t.is_string() && t.id != TypeId::Bool, SAILGPU_ERR_UNSUPPORTED, "min/max over " + t.str() + " is not supported on the GPU path yet");
    switch (x.kind) {
      case K_I32: return add_acc(is_min ? ACC_MIN_I32 : ACC_MAX_I32, &x);
      case K_I64: return add_acc(is_min ? ACC_MIN_I64 : ACC_MAX_I64, &x);
      case K_I128: return add_acc(is_min ? ACC_MIN_I128 : ACC_MAX_I128, &x);
      default: return add_acc(is_min ? ACC_MIN_F64 : ACC_MAX_F64, &x);
    }
  };

  // variance family: count, a double-double sum and a double-double sum of squares of the argument as Float64 (the count is the
  // argument's count|, shared with count / avg over it).  Merging, a state row's count is summed and its (count, mean, m2) feed
  // both sums: the sum reads the mean as its value, the sum of squares m2, and both the count and the mean (AccDesc::n_slot /
  // mean_slot).
  struct Moments { int jc, js, jq; };
  std::map<std::string, Val> as_f64;   // the argument as Float64, once per argument
  auto moments = [&](const Val& x0, const ExprPtr& x_expr, const DataType& t, const std::string& id, bool merge_rows) -> Moments {
    Moments m{};
    if (!merge_rows) {
      auto it = as_f64.find(id);
      if (it == as_f64.end()) {
        Val f;
        // a UInt64 lives in an I64 slot, which the cast would convert as signed
        if (t.id == TypeId::UInt64) { f = emit1(OP_CVT, K_F64, K_F64, x0, SRC_U64); f.vslot = x0.vslot; }
        else f = compile(make_cast(x_expr, T(TypeId::Float64)));
        it = as_f64.emplace(id, ensure_slot(f)).first;
      }
      const Val f = it->second;
      if (x0.vslot >= 0) { Val only_valid = x0; m.jc = add_acc(ACC_COUNT, &only_valid); } else m.jc = add_acc(ACC_COUNT, nullptr);
      ident("count|" + id, m.jc);
      m.js = ident("ddsum|" + id, add_acc(ACC_DD_SUM, &f));
      m.jq = ident("ddsq|" + id, add_acc(ACC_DD_SQ, &f));
      return m;
    }
    Val c = compile(bindings_.at(state_col_ + 0)), mean = compile(bindings_.at(state_col_ + 1)), m2 = compile(bindings_.at(state_col_ + 2));
    Val w = convert(c, K_I64); w.vslot = c.vslot;
    m.jc = ident("count|" + id, add_acc(ACC_SUM_I64, &w)); A.accs[m.jc].track_seen = 0;
    Val n = ensure_slot(convert(c, K_F64));
    Val mf = ensure_slot(convert(mean, K_F64)), qf = ensure_slot(convert(m2, K_F64));
    SG_CHECK(n.stride == 8 && mf.stride == 8, SAILGPU_ERR_INVALID, "variance state columns must be Float64");
    mf.vslot = c.vslot; qf.vslot = c.vslot;
    m.js = ident("ddsum|" + id, add_acc(ACC_DD_SUM, &mf));
    m.jq = ident("ddsq|" + id, add_acc(ACC_DD_SQ, &qf));
    for (int j : {m.js, m.jq}) { A.accs[j].n_slot = (uint32_t)n.slot; A.accs[j].mean_slot = (uint32_t)mf.slot; }
    return m;
  };

  // output columns: group keys first
  for (int i = 0; i < A.n_keys; ++i) {
    AggOutSpec o{}; o.kind = 0; o.a = i; o.b = key_first_word[(size_t)i]; o.type = key_types[(size_t)i]; o.nullable = A.keys[i].valid_slot != NO_SLOT;
    out.agg_outs.push_back(o);
  }
  size_t& state_col = state_col_;   // merging: cursor into the input state columns (current bindings)
  state_col = st.group_exprs.size();
  for (auto& a : st.aggs) {
    DataType in_t = a.input_type;
    Val arg; bool has_arg = false;
    std::string aid = "*";        // identity of the argument: its expression over the original input columns
    if (!merging && a.has_arg) { ExprPtr x = substitute(a.arg); arg = compile(x); in_t = x->type; has_arg = true; aid = x->key(); }
    if (merging) aid = "state" + std::to_string(state_col);
    SG_CHECK(a.fn == "count" || has_arg || merging, SAILGPU_ERR_INVALID, "aggregate '" + a.fn + "' needs an argument");
    AggTypes at = agg_types(a.fn, a.fn == "count" ? T(TypeId::Int64) : in_t);
    auto state_val = [&](size_t k) { return compile(bindings_.at(state_col + k)); };
    auto push_out = [&](int kind, int x, int y, const DataType& t, bool nullable) {
      AggOutSpec o{}; o.kind = kind; o.a = x; o.b = y; o.type = t; o.nullable = nullable; o.in_type = in_t;
      out.agg_outs.push_back(o);
    };
    Val xg;             // DISTINCT: the argument behind its gate
    if (a.distinct) { xg = ensure_slot(arg); xg.vslot = gate_for(arg, in_t, aid); }
    if (a.distinct && a.fn == "count") {
      push_out(1, ident("count|distinct|" + aid, add_acc(ACC_COUNT, &xg)), 0, T(TypeId::Int64), false);
    } else if (a.distinct && a.fn == "sum") {
      const int j = sum_acc(xg, in_t, "distinct|" + aid);
      push_out(1, j, 0, at.state[0], A.accs[j].track_seen != 0);
    } else if (a.distinct && a.fn == "avg") {
      const int jc = ident("count|distinct|" + aid, add_acc(ACC_COUNT, &xg));
      int js;
      if (in_t.is_decimal()) js = sum_acc(xg, in_t, "distinct|" + aid);
      else { Val f = convert(xg, K_F64); f.vslot = xg.vslot; js = ident("sumf|distinct|" + aid, add_acc(ACC_SUM_F64, &f)); }
      push_out(2, js, jc, at.final_type, true);
    } else if (a.fn == "count") {
      int j;
      if (merging) { Val s = state_val(0); Val w = convert(s, K_I64); w.vslot = s.vslot; j = add_acc(ACC_SUM_I64, &w); A.accs[j].track_seen = 0; }
      else if (has_arg && arg.vslot >= 0) { Val only_valid = arg; j = add_acc(ACC_COUNT, &only_valid); }
      else j = add_acc(ACC_COUNT, nullptr);
      ident("count|" + aid, j);
      push_out(1, j, 0, T(TypeId::Int64), false);
    } else if (a.fn == "sum") {
      Val x = merging ? state_val(0) : arg;
      int j = sum_acc(x, merging ? at.state[0] : in_t, aid);
      push_out(1, j, 0, at.state[0], A.accs[j].track_seen != 0);
    } else if (a.fn == "min" || a.fn == "max") {
      Val x = merging ? state_val(0) : arg;
      int j = ident(a.fn + "|" + aid, minmax_acc(a.fn == "min", x, in_t));
      push_out(1, j, 0, in_t, A.accs[j].track_seen != 0);
    } else if (a.fn == "avg") {
      int jc, js;
      if (merging) {
        Val c = state_val(0); Val w = convert(c, K_I64); w.vslot = c.vslot; jc = ident("count|" + aid, add_acc(ACC_SUM_I64, &w)); A.accs[jc].track_seen = 0;
        Val s = state_val(1);
        js = sum_acc(s, at.state[1], "state" + std::to_string(state_col + 1));
      } else {
        if (arg.vslot >= 0) { Val only_valid = arg; jc = add_acc(ACC_COUNT, &only_valid); } else jc = add_acc(ACC_COUNT, nullptr);
        ident("count|" + aid, jc);
        if (in_t.is_decimal()) js = sum_acc(arg, in_t, aid);
        else { Val f = convert(arg, K_F64); f.vslot = arg.vslot; js = ident("sumf|" + aid, add_acc(ACC_SUM_F64, &f)); }
      }
      if (partial) {
        push_out(1, jc, 0, T(TypeId::UInt64), false);
        push_out(1, js, 0, at.state[1], A.accs[js].track_seen != 0);
      } else {
        push_out(2, js, jc, at.final_type, true);
      }
    } else if (is_variance_fn(a.fn)) {
      const Moments mo = moments(arg, merging ? nullptr : substitute(a.arg), in_t, merging ? "state" + std::to_string(state_col) : aid, merging);
      if (partial) {
        push_out(1, mo.jc, 0, T(TypeId::UInt64), false);
        push_out(3, mo.js, mo.jc, T(TypeId::Float64), false);
        AggOutSpec o{}; o.kind = 4; o.a = mo.jq; o.b = mo.jc; o.c = mo.js; o.type = T(TypeId::Float64); o.nullable = false; o.in_type = in_t;
        out.agg_outs.push_back(o);
      } else {
        AggOutSpec o{}; o.kind = 5; o.a = mo.jq; o.b = mo.jc; o.c = mo.js; o.type = T(TypeId::Float64); o.nullable = true; o.in_type = in_t;
        o.var = variance_flags(a.fn);
        out.agg_outs.push_back(o);
      }
    } else fail(SAILGPU_ERR_UNSUPPORTED, "aggregate function '" + a.fn + "'");
    state_col += at.state.size();
  }
  {   // the extraction kernel takes at most MAX_KEYS + 2 * MAX_ACCS columns, in the operator's output and in the state rows
    size_t n_state = st.group_exprs.size();
    for (auto& a : st.aggs) n_state += agg_types(a.fn, a.fn == "count" ? T(TypeId::Int64) : a.input_type).state.size();
    SG_CHECK(std::max(out.agg_outs.size(), n_state) <= (size_t)(MAX_KEYS + 2 * MAX_ACCS), SAILGPU_ERR_UNSUPPORTED,
             "aggregate with more than " + std::to_string(MAX_KEYS + 2 * MAX_ACCS) + " output or state columns");
  }
  bool cas128 = false;
  for (int j = 0; j < A.n_accs; ++j) cas128 |= A.accs[j].op == ACC_MIN_I128 || A.accs[j].op == ACC_MAX_I128 || acc_is_dd(A.accs[j].op);
  if (cas128 && ((2 + A.key_words + words) & 1)) ++words;
  A.acc_words = words;
  A.entry_words = (uint32_t)(2 + A.key_words + A.acc_words);
  // integer fast path: every accumulator is a count or an integer/decimal sum without validity-dependent
  // NULL results, and few enough to live in registers
  {
    bool ok = A.n_accs <= REG_ACCS && getenv("SAILGPU_NO_REGPATH") == nullptr;
    for (int j = 0; j < A.n_accs; ++j) {
      const AccDesc& d = A.accs[j];
      ok &= (d.op == ACC_COUNT || d.op == ACC_SUM_I64 || d.op == ACC_SUM_I128) && !d.track_seen && d.valid_slot == NO_SLOT;
      ok &= d.op == ACC_COUNT || d.vkind == K_I64 || d.vkind == K_I128;
      ok &= !(d.op == ACC_SUM_I64 && d.vkind != K_I64);
    }
    A.reg_path = ok ? 1 : 0;
  }
  // word-wise key loading plan
  {
    int w = A.has_null_word;
    for (int i = 0; i < A.n_keys; ++i) {
      const KeyDesc& k = A.keys[i];
      const int nw = k.width == 16 ? 2 : 1;
      for (int q = 0; q < nw; ++q) {
        KeyWord kwd{}; kwd.slot = k.slot; kwd.valid_slot = k.valid_slot; kwd.stride = k.stride; kwd.key_index = (uint8_t)i;
        kwd.width = (uint8_t)(k.width == 16 ? 8 : k.width); kwd.byte_off = (uint8_t)(q * 8);
        A.kwords[w++] = kwd;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// layout: arena = [temps][hot scratch][stage 0 inputs][stage 1 inputs]
// ------------------------------------------------------------------------------------------------
static int env_int(const char* name, int dflt) { const char* v = getenv(name); return v && *v ? atoi(v) : dflt; }

void PipelineCompiler::finalize(CompiledPipeline& out, Ctx* ctx, int hot_wanted) {
  const size_t budget = ctx->max_smem;
  const size_t fixed = 256;
  SG_CHECK(prog_.size() <= (size_t)MAX_INST, SAILGPU_ERR_UNSUPPORTED, "fused pipeline needs more than " + std::to_string(MAX_INST) + " VM instructions");
  const AggParams& A = out.agg;
  if (out.sink != SINK_AGG || A.key_words > HOT_KEY_WORDS) hot_wanted = 0;
  auto layout = [&](int rpt, int stages, uint32_t* temps, uint32_t* stage) {
    const uint32_t tile = (uint32_t)rpt * NT;
    uint32_t t = 0, s = 0;
    for (auto& sl : slots_) {
      const uint32_t b = sl.bytes_per_row ? sl.bytes_per_row * tile : tile / 8;
      if (sl.is_input) s += (b + 127) & ~127u; else t += (b + 15) & ~15u;
    }
    *temps = (t + 127) & ~127u; *stage = s;
    return fixed + *temps + ((out.extra_scratch + 127) & ~127u) + (size_t)stages * s;
  };
  const int force_rpt = env_int("SAILGPU_RPT", 0), force_stages = env_int("SAILGPU_STAGES", 0), force_hot = env_int("SAILGPU_HOT", -1);
  // (rows per thread, input stages) in order of preference, as swept with scripts/sweep_q1.py and scripts/bench_ops.py (the
  // interpreter's order was tuned before the move to H100; the specialised kernel's stage count -- jit.cu: jit_plan -- was
  // measured on H100, DESIGN.md section 4.1):
  // aggregation wants 2 CTAs/SM of 512-row tiles; plain projection streams best with big double-buffered tiles;
  // compaction / join / partition sinks prefer big single-stage tiles and more resident CTAs
  static const int C_AGG[][2] = {{2, 1}, {1, 2}, {2, 2}, {1, 1}, {4, 1}, {4, 2}};
  // with the kernel specialiser on, dictionary aggregation uses 256-row tiles: the specialised kernel (which inherits the tile
  // size so that tile lists stay valid across both kernels) keeps one row per thread in registers without spills, which
  // beat two rows per thread on Q1; the interpreter, which now only sees small inputs, loses a few percent
  static const int C_AGG_JIT[][2] = {{1, 2}, {1, 1}, {2, 1}, {2, 2}, {4, 1}, {4, 2}};
  // high-cardinality aggregation is bound by the latency of the global table: small tiles, 4 CTAs/SM (64 registers)
  static const int C_AGG_COLD[][2] = {{2, 1}, {2, 2}, {1, 2}, {1, 1}, {4, 1}, {4, 2}};
  // the many-groups variant takes over the dictionary variant's deferred TILE list in the middle of a batch: same tile size
  static const int C_AGG_COLD_JIT[][2] = {{1, 2}, {1, 1}, {2, 1}, {2, 2}, {4, 1}, {4, 2}};
  static const int C_STORE[][2] = {{4, 2}, {4, 1}, {2, 2}, {2, 1}, {1, 2}, {1, 1}};
  static const int C_OTHER[][2] = {{4, 1}, {4, 2}, {2, 1}, {2, 2}, {1, 2}, {1, 1}};
  if (out.sink == SINK_AGG && out.cold_variant) hot_wanted = 0;
  // hash-join build and probe pipelines are bound by random-access latency as well (scripts/sweep_ops.sh: 5.4 vs 6.6 ms)
  const bool latency_bound = out.sink == SINK_BUILD || out.n_probes > 0;
  const bool jit_on = getenv("SAILGPU_JIT") == nullptr || atoi(getenv("SAILGPU_JIT")) != 0;
  const int (*cands)[2] = out.sink == SINK_AGG ? ((jit_on && out.n_probes == 0) ? (out.cold_variant ? C_AGG_COLD_JIT : C_AGG_JIT) : out.cold_variant ? C_AGG_COLD : C_AGG)
                          : out.sink == SINK_STORE ? C_STORE : latency_bound ? C_AGG_COLD : C_OTHER;
  int best_rpt = 0, best_stages = 0, best_hot = 0;
  if (hot_wanted > 0 && force_hot >= 0) hot_wanted = force_hot;
  hot_wanted = std::min(hot_wanted, HOT_MAX_GROUPS);
  for (int pass = 0; pass < 2 && !best_rpt; ++pass) {
    // pass 0: demand the wanted number of hot groups (min 4 when grouping); pass 1: whatever fits
    for (int ci = 0; ci < 6; ++ci) {
      const int* c = cands[ci];
      if (force_rpt && c[0] != force_rpt) continue;
      if (force_stages && c[1] != force_stages) continue;
      uint32_t t, s;
      const size_t need = layout(c[0], c[1], &t, &s);
      if (need > budget) continue;
      int hot = 0;       // the CTA dictionary takes what is left, up to hot_wanted groups
      while (hot < hot_wanted && need + hot_scratch_bytes(hot + 1, A.n_accs) <= budget) ++hot;
      if (pass == 0 && hot_wanted > 0 && hot < std::min(hot_wanted, 4)) continue;
      best_rpt = c[0]; best_stages = c[1]; best_hot = hot;
      break;
    }
  }
  SG_CHECK(best_rpt != 0, SAILGPU_ERR_UNSUPPORTED, "pipeline does not fit in shared memory (too many columns / temporaries)");
  out.rpt = best_rpt; out.n_stages = best_stages;
  uint32_t temps, stage;
  layout(best_rpt, best_stages, &temps, &stage);
  const uint32_t tile = (uint32_t)best_rpt * NT;
  out.temps_bytes = temps; out.stage_bytes = stage;
  out.hot_bytes = hot_scratch_bytes(best_hot, A.n_accs) + ((out.extra_scratch + 127) & ~127u);
  out.scratch_off = temps;
  // assign offsets
  uint32_t t_off = 0, s_off = temps + out.hot_bytes;
  for (auto& sl : slots_) {
    const uint32_t b = sl.bytes_per_row ? sl.bytes_per_row * tile : tile / 8;
    if (sl.is_input) { sl.offset = s_off | 0x80000000u; s_off += (b + 127) & ~127u; }
    else { sl.offset = t_off; t_off += (b + 15) & ~15u; }
  }
  out.arena_bytes = temps + out.hot_bytes + (uint32_t)best_stages * stage;
  out.smem_bytes = fixed + out.arena_bytes;
  {   // snapshot for the kernel specialiser, before ids become offsets
    JitInfo& J = out.jit;
    J.prog = prog_; J.slots = slots_; J.inputs = inputs_; J.mask = mask_;
    J.outs = out.outs; J.out_kinds = out_kinds_; J.agg = out.agg; J.keys = out.keys;
    for (int j = 0; j < MAX_ACCS; ++j) J.small_acc[j] = small_acc_[j];
    J.agg.hot_groups = best_hot;
    if (out.cold_variant) { J.agg.cold_only = 1; J.agg.reg_path = 0; }
    if (best_hot < REG_GROUPS) J.agg.reg_path = 0;
    J.valid = true;
  }
  auto off = [&](uint32_t id) -> uint32_t { return id == NO_SLOT ? NO_SLOT : slots_.at(id).offset; };
  out.prog = prog_;
  for (auto& I : out.prog) {
    I.dst = off(I.dst); I.a = off(I.a); I.b = off(I.b); I.c = off(I.c);
  }
  out.slots = slots_;
  out.inputs = inputs_;
  for (auto& in : out.inputs) in.slot = (int)off((uint32_t)in.slot);
  out.mask_slot = mask_.is_imm ? NO_SLOT : (mask_.slot >= 0 ? off((uint32_t)mask_.slot) : NO_SLOT);
  if (mask_.is_imm && mask_.i0 == 0) {
    // constant-false filter: materialise so that the sinks see an all-zero mask
    fail(SAILGPU_ERR_UNSUPPORTED, "constant FALSE predicate");
  }
  for (auto& o : out.outs) { o.slot = off(o.slot); o.valid_slot = off(o.valid_slot); }
  for (auto& k : out.keys) { k.slot = off(k.slot); k.valid_slot = off(k.valid_slot); }
  if (out.sink == SINK_AGG) {
    AggParams& AA = out.agg;
    for (int i = 0; i < AA.n_keys; ++i) { AA.keys[i].slot = off(AA.keys[i].slot); AA.keys[i].valid_slot = off(AA.keys[i].valid_slot); }
    for (int w = AA.has_null_word; w < AA.key_words; ++w) { AA.kwords[w].slot = off(AA.kwords[w].slot); AA.kwords[w].valid_slot = off(AA.kwords[w].valid_slot); }
    for (int j = 0; j < AA.n_accs; ++j) {
      AA.accs[j].value_slot = off(AA.accs[j].value_slot); AA.accs[j].valid_slot = off(AA.accs[j].valid_slot);
      AA.accs[j].n_slot = off(AA.accs[j].n_slot); AA.accs[j].mean_slot = off(AA.accs[j].mean_slot);
    }
    for (AggParams& D : out.distinct)
      for (int i = 0; i < D.n_keys; ++i) { D.keys[i].slot = off(D.keys[i].slot); D.keys[i].valid_slot = off(D.keys[i].valid_slot); }
    for (int j = 0; j < AA.n_accs && j < REG_ACCS; ++j) {
      AA.rload[j].slot = AA.accs[j].value_slot; AA.rload[j].stride = AA.accs[j].stride;
      AA.rload[j].mode = (uint8_t)(AA.accs[j].op == ACC_COUNT ? 0 : AA.accs[j].vkind == K_I64 ? (small_acc_[j] ? 3 : 1) : 2);
    }
    {
      bool simple = true;
      for (int w = 0; w < AA.key_words; ++w) simple &= !AA.has_null_word && AA.kwords[w].width == 8 && AA.kwords[w].valid_slot == NO_SLOT;
      AA.kw_simple = simple ? 1 : 0;
    }
    AA.hot_groups = best_hot;
    if (out.cold_variant) { AA.cold_only = 1; AA.reg_path = 0; }
    // the register fast path keeps its groups in the CTA dictionary: without one (keys wider than HOT_KEY_WORDS words,
    // or no shared memory left for it) every row has to take the general path
    if (AA.hot_groups < REG_GROUPS) AA.reg_path = 0;
    AA.hot_smem_off = temps;
  }
  for (ProbeParams* pp : probe_params) {
    for (int i = 0; i < pp->n_keys; ++i) { pp->keys[i].slot = off(pp->keys[i].slot); pp->keys[i].valid_slot = off(pp->keys[i].valid_slot); }
    pp->match_slot = off(pp->match_slot); pp->rowid_slot = off(pp->rowid_slot);
  }
  out.literals = literals_;
  out.literal_fixups = literal_fixups_;
}

}  // namespace sg
