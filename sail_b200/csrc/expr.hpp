// expr.hpp -- physical expressions: parsing from the JSON spec and DataFusion/arrow-rs type rules.
//
// Mirrors what Sail hands DataFusion after planning: BinaryExpr / Literal / Column / CastExpr /
// CaseExpr / InListExpr / LikeExpr / NotExpr / IsNull / ScalarFunction(date_part, date_trunc, substr, character_length)
// (crates/sail-plan/src/function/scalar/math.rs:48-181,580-583; predicate.rs:103-125).
// Result types follow arrow-arith 58 (SURVEY.md Appendix A).
#pragma once
#include <algorithm>

#include "common.hpp"
#include "vm.h"

namespace sg {

struct Expr;
using ExprPtr = std::shared_ptr<Expr>;

struct Expr {
  enum Kind { Col, Lit, Bin, Not, Neg, IsNull, IsNotNull, Cast, Case, Like, DatePart, Substr, DateTrunc, CharLength } kind = Col;
  DataType type;
  bool nullable = false;
  // Col
  int col = -1;
  // Lit
  bool lit_null = false;
  i128 lit_i = 0;        // ints, decimals (unscaled), dates, bools
  double lit_f = 0.0;
  std::string lit_s;
  // Bin / Like / DatePart
  std::string op;        // "+", "=", "and", ... ; LIKE pattern ; date part
  bool negated = false;
  long long sub_start = 1, sub_len = -1;     // Substr: 1-based first character, character count (-1: to the end)
  std::vector<ExprPtr> args;   // Bin: l, r ; Case: w0,t0,w1,t1,...,[else]
  bool has_else = false;

  std::string key() const;     // structural key for common-subexpression elimination
};

inline std::string i128_str(i128 v) {
  if (v == 0) return "0";
  bool neg = v < 0; u128 u = neg ? (u128)0 - (u128)v : (u128)v; std::string s;
  while (u) { s += (char)('0' + (int)(u % 10)); u /= 10; }
  if (neg) s += '-';
  std::reverse(s.begin(), s.end());
  return s;
}

inline std::string Expr::key() const {
  switch (kind) {
    case Col: return "c" + std::to_string(col);
    case Lit: return "l[" + type.str() + ":" + (lit_null ? "null" : type.is_string() ? lit_s : type.is_float() ? std::to_string(lit_f) : i128_str(lit_i)) + "]";
    default: {
      std::string s = std::to_string((int)kind) + "(" + op + (negated ? "!" : "") + ":" + type.str();
      for (auto& a : args) s += "," + a->key();
      return s + ")";
    }
  }
}

inline DataType int_as_decimal(const DataType& t) {
  switch (t.id) {
    case TypeId::Int8: case TypeId::UInt8: return Dec(3, 0);
    case TypeId::Int16: case TypeId::UInt16: return Dec(5, 0);
    case TypeId::Int32: case TypeId::UInt32: return Dec(10, 0);
    default: return Dec(20, 0);
  }
}

inline DataType decimal_result(const std::string& op, const DataType& a, const DataType& b) {
  int p1 = a.precision, s1 = a.scale, p2 = b.precision, s2 = b.scale;
  if (op == "+" || op == "-") { int s = std::max(s1, s2); return Dec(std::min(38, std::max(p1 - s1, p2 - s2) + s + 1), s); }
  if (op == "*") return Dec(std::min(38, p1 + p2 + 1), s1 + s2);
  if (op == "/") { int s = std::min(38, s1 + 4); return Dec(std::min(38, p1 - s1 + s2 + s), s); }
  if (op == "%") { int s = std::max(s1, s2); return Dec(std::min(38, std::min(p1 - s1, p2 - s2) + s), s); }
  fail(SAILGPU_ERR_INVALID, "bad decimal op " + op);
}

// Casts that involve a Timestamp (arrow-rs semantics): Int64 <-> Timestamp reinterpret the value, Timestamp -> Date32 takes the
// local date in the column's zone, Timestamp -> Timestamp of the same or a finer unit multiplies.  Everything else is refused.
inline void check_timestamp_cast(const DataType& from, const DataType& to) {
  if (!from.is_timestamp() && !to.is_timestamp()) return;
  const std::string what = "cast " + from.str() + " -> " + to.str();
  if (from.is_timestamp() && to.is_timestamp()) {
    SG_CHECK(to.unit >= from.unit, SAILGPU_ERR_UNSUPPORTED, what + " (to a coarser unit) is not supported on the GPU path");
    // between two zones the instant is kept; adding or dropping a zone would reinterpret wall-clock time
    SG_CHECK(from.tz == to.tz || (!from.tz.empty() && !to.tz.empty()), SAILGPU_ERR_UNSUPPORTED, what + " is not supported on the GPU path");
    return;
  }
  if (from.is_timestamp() && to.id == TypeId::Date32) { zone_offset_seconds(from.tz); return; }
  SG_CHECK((from.is_timestamp() && to.id == TypeId::Int64) || (to.is_timestamp() && from.id == TypeId::Int64), SAILGPU_ERR_UNSUPPORTED,
           what + " is not supported on the GPU path");
}

// Every cast, explicit or implied (CASE branches brought to one type, operand coercion), is built here, so the Timestamp
// rules hold for all of them.
inline ExprPtr make_cast(ExprPtr e, const DataType& to) {
  if (e->type == to) return e;
  check_timestamp_cast(e->type, to);
  auto c = std::make_shared<Expr>();
  c->kind = Expr::Cast; c->type = to; c->nullable = e->nullable; c->args = {e};
  return c;
}

// date_part / date_trunc parts on a Timestamp (vm.h: TsPart); -1 = not a part of `fn`
inline int timestamp_part(const std::string& fn, const std::string& part) {
  static const char* names[] = {"year", "quarter", "month", "week", "day", "hour", "minute", "second"};
  for (int k = TS_YEAR; k <= TS_SECOND; ++k)
    if (part == names[k]) return fn == "date_part" && k == TS_WEEK ? -1 : k;
  return -1;
}

inline bool is_arith(const std::string& op) { return op == "+" || op == "-" || op == "*" || op == "/" || op == "%"; }
inline bool is_cmp(const std::string& op) { return op == "=" || op == "!=" || op == "<" || op == "<=" || op == ">" || op == ">="; }

// numeric coercion for operands that arrive with different types (plans normally arrive coerced)
inline void coerce_numeric(ExprPtr& l, ExprPtr& r, bool for_compare) {
  const DataType a = l->type, b = r->type;
  if (a == b) return;
  if (a.is_decimal() && b.is_int()) { r = make_cast(r, int_as_decimal(b)); }
  else if (b.is_decimal() && a.is_int()) { l = make_cast(l, int_as_decimal(a)); }
  else if (a.is_float() || b.is_float()) { l = make_cast(l, T(TypeId::Float64)); r = make_cast(r, T(TypeId::Float64)); }
  else if (a.is_int() && b.is_int()) { l = make_cast(l, T(TypeId::Int64)); r = make_cast(r, T(TypeId::Int64)); }
  if (for_compare && l->type.is_decimal() && r->type.is_decimal() && l->type != r->type) {
    // compare at the wider scale / integer-digit count
    int s = std::max(l->type.scale, r->type.scale);
    int ip = std::max(l->type.precision - l->type.scale, r->type.precision - r->type.scale);
    DataType t = Dec(std::min(38, ip + s), s);
    l = make_cast(l, t); r = make_cast(r, t);
  }
}

ExprPtr parse_expr(const Json& j, const Schema& in);

inline ExprPtr parse_literal(const Json& j) {
  auto e = std::make_shared<Expr>();
  e->kind = Expr::Lit;
  e->type = parse_type(j.at("type").as_str());
  const Json& v = j.at("lit");
  if (v.is_null()) { e->lit_null = true; e->nullable = true; return e; }
  if (e->type.is_string()) e->lit_s = v.as_str();
  else if (e->type.is_float()) e->lit_f = v.as_double();
  else if (e->type.id == TypeId::Bool) e->lit_i = v.kind == Json::Bool ? (v.b ? 1 : 0) : (v.as_int() != 0);
  else e->lit_i = parse_i128(v.s);
  return e;
}

inline ExprPtr make_bin(const std::string& op, ExprPtr l, ExprPtr r) {
  auto e = std::make_shared<Expr>();
  e->kind = Expr::Bin; e->op = op;
  if (is_arith(op)) {
    coerce_numeric(l, r, false);
    if (l->type.is_decimal() && r->type.is_decimal()) e->type = decimal_result(op, l->type, r->type);
    else {
      SG_CHECK(l->type == r->type, SAILGPU_ERR_UNSUPPORTED, "arithmetic on " + l->type.str() + " and " + r->type.str());
      SG_CHECK(l->type.is_int() || l->type.is_float(), SAILGPU_ERR_UNSUPPORTED, "arithmetic on " + l->type.str());
      e->type = l->type;
    }
  } else if (is_cmp(op)) {
    if (l->type.is_timestamp() || r->type.is_timestamp()) {
      // instants compare across zones; across units they would need a rescale, which DataFusion's coercion adds as a cast
      SG_CHECK(l->type.is_timestamp() && r->type.is_timestamp() && l->type.unit == r->type.unit, SAILGPU_ERR_UNSUPPORTED,
               "comparison of " + l->type.str() + " and " + r->type.str());
    } else if (l->type.is_string() && r->type.is_string()) {
      SG_CHECK(op == "=" || op == "!=", SAILGPU_ERR_UNSUPPORTED, "ordering comparison on strings is not supported on the GPU path yet");
    } else {
      coerce_numeric(l, r, true);
      SG_CHECK(l->type == r->type, SAILGPU_ERR_UNSUPPORTED, "comparison of " + l->type.str() + " and " + r->type.str());
    }
    e->type = T(TypeId::Bool);
  } else if (op == "and" || op == "or") {
    SG_CHECK(l->type.id == TypeId::Bool && r->type.id == TypeId::Bool, SAILGPU_ERR_INVALID, "AND/OR need boolean operands");
    e->type = T(TypeId::Bool);
  } else {
    fail(SAILGPU_ERR_UNSUPPORTED, "binary operator '" + op + "'");
  }
  e->nullable = l->nullable || r->nullable;
  e->args = {l, r};
  return e;
}

inline ExprPtr parse_expr(const Json& j, const Schema& in) {
  SG_CHECK(j.kind == Json::Obj, SAILGPU_ERR_INVALID, "spec: expression must be an object");
  if (j.has("col")) {
    auto e = std::make_shared<Expr>();
    int c = (int)j.at("col").as_int();
    SG_CHECK(c >= 0 && c < (int)in.size(), SAILGPU_ERR_INVALID, "spec: column index " + std::to_string(c) + " out of range");
    e->kind = Expr::Col; e->col = c; e->type = in[c].type; e->nullable = in[c].nullable;
    return e;
  }
  if (j.has("lit")) return parse_literal(j);
  if (j.has("op")) return make_bin(j.at("op").as_str(), parse_expr(j.at("l"), in), parse_expr(j.at("r"), in));
  auto e = std::make_shared<Expr>();
  if (j.has("not")) {
    e->kind = Expr::Not; e->args = {parse_expr(j.at("not"), in)}; e->type = T(TypeId::Bool); e->nullable = e->args[0]->nullable;
    SG_CHECK(e->args[0]->type.id == TypeId::Bool, SAILGPU_ERR_INVALID, "NOT needs a boolean operand");
    return e;
  }
  if (j.has("neg")) {
    e->kind = Expr::Neg; e->args = {parse_expr(j.at("neg"), in)}; e->type = e->args[0]->type; e->nullable = e->args[0]->nullable;
    SG_CHECK(!e->type.is_timestamp(), SAILGPU_ERR_UNSUPPORTED, "negation of " + e->type.str());
    return e;
  }
  if (j.has("is_null") || j.has("is_not_null")) {
    const bool isn = j.has("is_null");
    e->kind = isn ? Expr::IsNull : Expr::IsNotNull;
    e->args = {parse_expr(j.at(isn ? "is_null" : "is_not_null"), in)}; e->type = T(TypeId::Bool);
    return e;
  }
  if (j.has("cast")) return make_cast(parse_expr(j.at("cast"), in), parse_type(j.at("to").as_str()));
  if (j.has("case")) {
    e->kind = Expr::Case;
    std::vector<ExprPtr> thens;
    for (auto& br : j.at("case").a) {
      SG_CHECK(br.kind == Json::Arr && br.a.size() == 2, SAILGPU_ERR_INVALID, "spec: CASE branch must be [when, then]");
      e->args.push_back(parse_expr(br.a[0], in));
      e->args.push_back(parse_expr(br.a[1], in));
      thens.push_back(e->args.back());
    }
    const Json* el = j.find("else");
    ExprPtr els;
    if (el && !el->is_null()) { els = parse_expr(*el, in); thens.push_back(els); }
    DataType rt = thens[0]->type;
    bool alldec = true; for (auto& t : thens) alldec &= t->type.is_decimal();
    if (alldec) {
      int s = 0, ip = 0;
      for (auto& t : thens) { s = std::max(s, t->type.scale); ip = std::max(ip, t->type.precision - t->type.scale); }
      rt = Dec(std::min(38, ip + s), s);
    }
    for (size_t i = 1; i < e->args.size(); i += 2) e->args[i] = make_cast(e->args[i], rt);
    e->nullable = !els;
    for (size_t i = 1; i < e->args.size(); i += 2) e->nullable |= e->args[i]->nullable;
    if (els) { els = make_cast(els, rt); e->nullable |= els->nullable; e->args.push_back(els); e->has_else = true; }
    e->type = rt;
    return e;
  }
  if (j.has("in")) {
    // InListExpr over literals == OR of equalities (NULL semantics identical for non-null lists)
    ExprPtr x = parse_expr(j.at("in"), in), acc;
    for (auto& l : j.at("set").a) {
      ExprPtr eq = make_bin("=", x, parse_literal(l));
      acc = acc ? make_bin("or", acc, eq) : eq;
    }
    SG_CHECK((bool)acc, SAILGPU_ERR_INVALID, "spec: empty IN list");
    const Json* neg = j.find("negated");
    if (neg && neg->kind == Json::Bool && neg->b) {
      auto n = std::make_shared<Expr>();
      n->kind = Expr::Not; n->args = {acc}; n->type = T(TypeId::Bool); n->nullable = acc->nullable;
      return n;
    }
    return acc;
  }
  if (j.has("like")) {
    e->kind = Expr::Like; e->args = {parse_expr(j.at("like"), in)}; e->op = j.at("pattern").as_str();
    const Json* neg = j.find("negated"); e->negated = neg && neg->kind == Json::Bool && neg->b;
    SG_CHECK(e->args[0]->type.is_string(), SAILGPU_ERR_INVALID, "LIKE needs a string operand");
    e->type = T(TypeId::Bool); e->nullable = e->args[0]->nullable;
    return e;
  }
  if (j.has("fn")) {
    const std::string fn = j.at("fn").as_str();
    if (fn == "date_part" || fn == "date_trunc") {
      // On a Timestamp: the part in the column's zone (date_part: Int32, second as Decimal128(8,6) like Spark's; date_trunc: the
      // input's type).  On a Date32: date_part of year, month or day, as Int32.
      ExprPtr x = parse_expr(j.at("args").a.at(0), in);
      std::string part = j.at("part").as_str();
      std::transform(part.begin(), part.end(), part.begin(), ::tolower);
      e->op = part; e->args = {x}; e->nullable = x->nullable;
      if (x->type.is_timestamp()) {
        const int k = timestamp_part(fn, part);
        SG_CHECK(k >= 0, SAILGPU_ERR_UNSUPPORTED, fn + "('" + part + "') on " + x->type.str());
        zone_offset_seconds(x->type.tz);
        e->kind = fn == "date_part" ? Expr::DatePart : Expr::DateTrunc;
        e->type = fn == "date_trunc" ? x->type : k == TS_SECOND ? Dec(8, 6) : T(TypeId::Int32);
        return e;
      }
      SG_CHECK(fn == "date_part", SAILGPU_ERR_UNSUPPORTED, "date_trunc on " + x->type.str());
      SG_CHECK(part == "year" || part == "month" || part == "day", SAILGPU_ERR_UNSUPPORTED, "date_part('" + part + "')");
      SG_CHECK(x->type.id == TypeId::Date32, SAILGPU_ERR_UNSUPPORTED, "date_part on " + x->type.str());
      e->kind = Expr::DatePart; e->type = T(TypeId::Int32);
      return e;
    }
    if (fn == "substr") {      // substr(str, start[, length]) with literal positions (Spark / DataFusion character semantics)
      e->kind = Expr::Substr;
      e->args = {parse_expr(j.at("args").a.at(0), in)};
      SG_CHECK(e->args[0]->type.is_string(), SAILGPU_ERR_INVALID, "substr needs a string operand");
      e->sub_start = j.at("start").as_int();
      const Json* ln = j.find("length");
      e->sub_len = ln && !ln->is_null() ? ln->as_int() : -1;
      SG_CHECK(e->sub_start >= 1, SAILGPU_ERR_UNSUPPORTED, "substr with a start position below 1 is not supported on the GPU path yet");
      SG_CHECK(!(ln && !ln->is_null()) || e->sub_len >= 0, SAILGPU_ERR_INVALID, "substr with a negative length");
      e->op = "substr:" + std::to_string(e->sub_start) + ":" + std::to_string(e->sub_len);
      e->type = e->args[0]->type; e->nullable = e->args[0]->nullable;
      return e;
    }
    if (fn == "character_length") {      // characters of a Utf8 / Utf8View string as Int32, DataFusion's type for both
      e->kind = Expr::CharLength;
      SG_CHECK(j.at("args").a.size() == 1, SAILGPU_ERR_INVALID, "character_length takes one argument");
      e->args = {parse_expr(j.at("args").a[0], in)};
      SG_CHECK(e->args[0]->type.is_string(), SAILGPU_ERR_INVALID, "character_length needs a string operand");
      e->type = T(TypeId::Int32); e->nullable = e->args[0]->nullable;
      return e;
    }
    fail(SAILGPU_ERR_UNSUPPORTED, "scalar function '" + fn + "' is not implemented on the GPU path");
  }
  fail(SAILGPU_ERR_INVALID, "spec: unrecognised expression object");
}

// ---- aggregate typing (DataFusion UDAFs; SURVEY.md Appendix A) ------------------------------------
// The variance family under the names DataFusion's physical plan gives its UDAFs: stddev and var are the sample forms.
inline bool is_variance_fn(const std::string& fn) { return fn == "stddev" || fn == "stddev_pop" || fn == "var" || fn == "var_pop"; }
inline int variance_flags(const std::string& fn) {
  return (fn == "stddev_pop" || fn == "var_pop" ? VAR_POP : 0) | (fn == "stddev" || fn == "stddev_pop" ? VAR_SQRT : 0);
}
struct AggTypes { std::vector<DataType> state; DataType final_type; };
inline AggTypes agg_types(const std::string& fn, const DataType& in) {
  AggTypes t;
  if (fn == "count") { t.state = {T(TypeId::Int64)}; t.final_type = T(TypeId::Int64); return t; }
  if (fn == "min" || fn == "max") { t.state = {in}; t.final_type = in; return t; }
  SG_CHECK(!in.is_timestamp(), SAILGPU_ERR_UNSUPPORTED, fn + " over " + in.str());
  if (fn == "sum") {
    DataType s = in.is_decimal() ? Dec(std::min(38, in.precision + 10), in.scale)
               : in.is_float() ? T(TypeId::Float64) : in.is_unsigned_int() ? T(TypeId::UInt64) : T(TypeId::Int64);
    t.state = {s}; t.final_type = s; return t;
  }
  if (fn == "avg") {
    if (in.is_decimal()) {
      t.state = {T(TypeId::UInt64), Dec(std::min(38, in.precision + 10), in.scale)};
      t.final_type = Dec(std::min(38, in.precision + 4), std::min(38, in.scale + 4));
    } else {
      t.state = {T(TypeId::UInt64), T(TypeId::Float64)};
      t.final_type = T(TypeId::Float64);
    }
    return t;
  }
  if (is_variance_fn(fn)) {
    // DataFusion coerces the argument to Float64; its state is the count, mean and sum of squared deviations
    SG_CHECK(in.is_int() || in.is_decimal() || in.is_float(), SAILGPU_ERR_INVALID, fn + " over " + in.str());
    t.state = {T(TypeId::UInt64), T(TypeId::Float64), T(TypeId::Float64)};
    t.final_type = T(TypeId::Float64);
    return t;
  }
  fail(SAILGPU_ERR_UNSUPPORTED, "aggregate function '" + fn + "'");
}

}  // namespace sg
