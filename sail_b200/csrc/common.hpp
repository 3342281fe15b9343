// common.hpp -- errors, data types and a minimal JSON reader shared by the host side of libsailgpu.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/sailgpu.h"

namespace sg {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
[[noreturn]] inline void fail(int code, const std::string& m) { throw Error(code, m); }
#define SG_CHECK(cond, code, msg) \
  do { if (!(cond)) ::sg::fail((code), (msg)); } while (0)

// ------------------------------------------------------------------------------------------------
// Data types (the subset of Arrow types Sail's TPC-H / ClickBench plans put on the hot path)
// ------------------------------------------------------------------------------------------------
enum class TypeId : uint8_t {
  Bool, Int8, Int16, Int32, Int64, UInt8, UInt16, UInt32, UInt64, Float32, Float64, Date32,
  Decimal128, Utf8, Utf8View, Timestamp, Null
};

enum TimeUnit : int { TU_S = 0, TU_MS = 1, TU_US = 2, TU_NS = 3 };
inline int64_t unit_per_second(int unit) { return unit == TU_S ? 1 : unit == TU_MS ? 1000 : unit == TU_US ? 1000000 : 1000000000; }

struct DataType {
  TypeId id = TypeId::Null;
  int precision = 0, scale = 0;
  int unit = TU_S;        // Timestamp: TimeUnit
  std::string tz;         // Timestamp: zone as Arrow carries it ("" = none)
  bool operator==(const DataType& o) const {
    return id == o.id && precision == o.precision && scale == o.scale && unit == o.unit && tz == o.tz;
  }
  bool operator!=(const DataType& o) const { return !(*this == o); }
  bool is_timestamp() const { return id == TypeId::Timestamp; }
  // How values are laid out and compared on the device.  A Timestamp is stored as Int64 (Arrow's layout); everything that
  // moves, hashes, compares or accumulates values asks for this type, so only expressions that read wall-clock time know
  // the Timestamp type itself.
  DataType storage() const;
  bool is_decimal() const { return id == TypeId::Decimal128; }
  bool is_string() const { return id == TypeId::Utf8 || id == TypeId::Utf8View; }
  bool is_float() const { return id == TypeId::Float32 || id == TypeId::Float64; }
  bool is_signed_int() const { return id == TypeId::Int8 || id == TypeId::Int16 || id == TypeId::Int32 || id == TypeId::Int64; }
  bool is_unsigned_int() const { return id == TypeId::UInt8 || id == TypeId::UInt16 || id == TypeId::UInt32 || id == TypeId::UInt64; }
  bool is_int() const { return is_signed_int() || is_unsigned_int(); }
  // bytes per value in the Arrow values buffer (Bool is bit-packed -> 0; Utf8 offsets -> 4)
  int arrow_width() const {
    switch (id) {
      case TypeId::Bool: return 0;
      case TypeId::Int8: case TypeId::UInt8: return 1;
      case TypeId::Int16: case TypeId::UInt16: return 2;
      case TypeId::Int32: case TypeId::UInt32: case TypeId::Float32: case TypeId::Date32: return 4;
      case TypeId::Int64: case TypeId::UInt64: case TypeId::Float64: case TypeId::Timestamp: return 8;
      case TypeId::Decimal128: case TypeId::Utf8View: return 16;
      case TypeId::Utf8: return 4;
      default: return 0;
    }
  }
  std::string str() const;
  std::string arrow_format() const;  // Arrow C data interface format string
};

inline DataType T(TypeId id) { DataType t; t.id = id; return t; }
inline DataType Dec(int p, int s) { DataType t; t.id = TypeId::Decimal128; t.precision = p; t.scale = s; return t; }
inline DataType Ts(int unit, const std::string& tz) { DataType t; t.id = TypeId::Timestamp; t.unit = unit; t.tz = tz; return t; }
inline DataType DataType::storage() const { return id == TypeId::Timestamp ? T(TypeId::Int64) : *this; }

inline const char* unit_name(int unit) { return unit == TU_S ? "s" : unit == TU_MS ? "ms" : unit == TU_US ? "us" : "ns"; }

// Zone of a Timestamp as the functions that read wall-clock time need it: the offset from UTC in seconds.  Accepted: no zone,
// "UTC", and fixed offsets "+HH:MM" / "-HH:MM".  Anything else (an IANA name such as "Europe/Paris") needs a time-zone
// database and is refused.
inline int64_t zone_offset_seconds(const std::string& tz) {
  if (tz.empty() || tz == "UTC") return 0;
  int hh = 0, mm = 0;
  char sign = 0, colon = 0;
  if (tz.size() == 6 && sscanf(tz.c_str(), "%c%2d%c%2d", &sign, &hh, &colon, &mm) == 4 && (sign == '+' || sign == '-') && colon == ':' &&
      isdigit((unsigned char)tz[1]) && isdigit((unsigned char)tz[2]) && isdigit((unsigned char)tz[4]) && isdigit((unsigned char)tz[5]) &&
      hh <= 23 && mm <= 59)
    return (sign == '-' ? -1 : 1) * (int64_t)(hh * 3600 + mm * 60);
  fail(SAILGPU_ERR_UNSUPPORTED, "time zone '" + tz + "' is not supported on the GPU path (only UTC and fixed offsets +HH:MM)");
}

inline std::string DataType::str() const {
  switch (id) {
    case TypeId::Bool: return "Boolean";
    case TypeId::Int8: return "Int8"; case TypeId::Int16: return "Int16";
    case TypeId::Int32: return "Int32"; case TypeId::Int64: return "Int64";
    case TypeId::UInt8: return "UInt8"; case TypeId::UInt16: return "UInt16";
    case TypeId::UInt32: return "UInt32"; case TypeId::UInt64: return "UInt64";
    case TypeId::Float32: return "Float32"; case TypeId::Float64: return "Float64";
    case TypeId::Date32: return "Date32";
    case TypeId::Decimal128: return "Decimal128(" + std::to_string(precision) + "," + std::to_string(scale) + ")";
    case TypeId::Utf8: return "Utf8"; case TypeId::Utf8View: return "Utf8View";
    case TypeId::Timestamp: return std::string("Timestamp(") + unit_name(unit) + (tz.empty() ? "" : ", " + tz) + ")";
    default: return "Null";
  }
}
inline std::string DataType::arrow_format() const {
  switch (id) {
    case TypeId::Bool: return "b";
    case TypeId::Int8: return "c"; case TypeId::UInt8: return "C";
    case TypeId::Int16: return "s"; case TypeId::UInt16: return "S";
    case TypeId::Int32: return "i"; case TypeId::UInt32: return "I";
    case TypeId::Int64: return "l"; case TypeId::UInt64: return "L";
    case TypeId::Float32: return "f"; case TypeId::Float64: return "g";
    case TypeId::Date32: return "tdD";
    case TypeId::Decimal128: return "d:" + std::to_string(precision) + "," + std::to_string(scale);
    case TypeId::Utf8: return "u"; case TypeId::Utf8View: return "vu";
    case TypeId::Timestamp: return std::string("ts") + "smun"[unit] + ":" + tz;
    default: return "n";
  }
}
inline DataType parse_type(const std::string& s) {
  static const std::map<std::string, TypeId> m = {
      {"Boolean", TypeId::Bool}, {"Int8", TypeId::Int8}, {"Int16", TypeId::Int16}, {"Int32", TypeId::Int32},
      {"Int64", TypeId::Int64}, {"UInt8", TypeId::UInt8}, {"UInt16", TypeId::UInt16}, {"UInt32", TypeId::UInt32},
      {"UInt64", TypeId::UInt64}, {"Float32", TypeId::Float32}, {"Float64", TypeId::Float64},
      {"Date32", TypeId::Date32}, {"Utf8", TypeId::Utf8}, {"Utf8View", TypeId::Utf8View}};
  auto it = m.find(s);
  if (it != m.end()) return T(it->second);
  int p = 0, sc = 0;
  if (sscanf(s.c_str(), "Decimal128(%d,%d)", &p, &sc) == 2 || sscanf(s.c_str(), "Decimal128(%d, %d)", &p, &sc) == 2)
    return Dec(p, sc);
  if (s.size() > 11 && s.compare(0, 10, "Timestamp(") == 0 && s.back() == ')') {   // Timestamp(<unit>[, <zone>])
    std::string body = s.substr(10, s.size() - 11), u = body, tz;
    const size_t comma = body.find(',');
    if (comma != std::string::npos) {
      u = body.substr(0, comma);
      tz = body.substr(comma + 1);
      while (!tz.empty() && tz.front() == ' ') tz.erase(0, 1);
    }
    for (int k = TU_S; k <= TU_NS; ++k)
      if (u == unit_name(k)) return Ts(k, tz);
  }
  fail(SAILGPU_ERR_UNSUPPORTED, "unsupported data type '" + s + "'");
}
inline DataType type_from_arrow_format(const char* f) {
  std::string s(f);
  if (s == "b") return T(TypeId::Bool);
  if (s == "c") return T(TypeId::Int8); if (s == "C") return T(TypeId::UInt8);
  if (s == "s") return T(TypeId::Int16); if (s == "S") return T(TypeId::UInt16);
  if (s == "i") return T(TypeId::Int32); if (s == "I") return T(TypeId::UInt32);
  if (s == "l") return T(TypeId::Int64); if (s == "L") return T(TypeId::UInt64);
  if (s == "f") return T(TypeId::Float32); if (s == "g") return T(TypeId::Float64);
  if (s == "tdD") return T(TypeId::Date32);
  if (s == "u") return T(TypeId::Utf8); if (s == "vu") return T(TypeId::Utf8View);
  if (s.size() >= 4 && s[0] == 't' && s[1] == 's' && s[3] == ':') {   // tss: / tsm: / tsu: / tsn: followed by the zone (may be empty)
    const char* units = "smun";
    const char* u = strchr(units, s[2]);
    if (s[2] && u) return Ts((int)(u - units), s.substr(4));
  }
  int p = 0, sc = 0, bits = 128;
  if (sscanf(f, "d:%d,%d,%d", &p, &sc, &bits) >= 2) {
    SG_CHECK(bits == 128, SAILGPU_ERR_UNSUPPORTED, "only 128-bit decimals are supported");
    return Dec(p, sc);
  }
  fail(SAILGPU_ERR_UNSUPPORTED, "unsupported Arrow format '" + s + "'");
}

struct Field { std::string name; DataType type; bool nullable = true; };
using Schema = std::vector<Field>;

// ------------------------------------------------------------------------------------------------
// minimal JSON (objects, arrays, strings, numbers, true/false/null) -- enough for operator specs
// ------------------------------------------------------------------------------------------------
struct Json {
  enum Kind { Null, Bool, Num, Str, Arr, Obj } kind = Null;
  bool b = false;
  std::string s;     // Str, and the raw text of Num (so 128-bit integers survive)
  std::vector<Json> a;
  std::vector<std::pair<std::string, Json>> o;

  bool is_null() const { return kind == Null; }
  bool has(const char* k) const {
    for (auto& kv : o) if (kv.first == k) return true;
    return false;
  }
  const Json& at(const char* k) const {
    for (auto& kv : o) if (kv.first == k) return kv.second;
    fail(SAILGPU_ERR_INVALID, std::string("spec: missing key '") + k + "'");
  }
  const Json* find(const char* k) const {
    for (auto& kv : o) if (kv.first == k) return &kv.second;
    return nullptr;
  }
  int64_t as_int() const {
    SG_CHECK(kind == Num || kind == Str, SAILGPU_ERR_INVALID, "spec: expected integer");
    return strtoll(s.c_str(), nullptr, 10);
  }
  double as_double() const {
    SG_CHECK(kind == Num || kind == Str, SAILGPU_ERR_INVALID, "spec: expected number");
    return strtod(s.c_str(), nullptr);
  }
  bool as_bool() const { SG_CHECK(kind == Bool, SAILGPU_ERR_INVALID, "spec: expected bool"); return b; }
  const std::string& as_str() const { SG_CHECK(kind == Str, SAILGPU_ERR_INVALID, "spec: expected string"); return s; }
};
// canonical text of a spec (cache keys)
inline void json_dump(const Json& j, std::string* out) {
  switch (j.kind) {
    case Json::Null: *out += "null"; break;
    case Json::Bool: *out += j.b ? "true" : "false"; break;
    case Json::Num: *out += j.s; break;
    case Json::Str: *out += '"'; *out += j.s; *out += '"'; break;
    case Json::Arr: *out += '['; for (auto& x : j.a) { json_dump(x, out); *out += ','; } *out += ']'; break;
    case Json::Obj: *out += '{'; for (auto& kv : j.o) { *out += kv.first; *out += ':'; json_dump(kv.second, out); *out += ','; } *out += '}'; break;
  }
}


class JsonParser {
 public:
  JsonParser(const char* p, size_t n) : p_(p), e_(p + n) {}
  Json parse() { Json j = value(); ws(); SG_CHECK(p_ == e_, SAILGPU_ERR_INVALID, "spec: trailing characters"); return j; }
 private:
  const char *p_, *e_;
  void ws() { while (p_ < e_ && (*p_ == ' ' || *p_ == '\n' || *p_ == '\t' || *p_ == '\r')) ++p_; }
  char peek() { ws(); SG_CHECK(p_ < e_, SAILGPU_ERR_INVALID, "spec: unexpected end"); return *p_; }
  void expect(char c) { SG_CHECK(peek() == c, SAILGPU_ERR_INVALID, std::string("spec: expected '") + c + "'"); ++p_; }
  Json value() {
    char c = peek();
    Json j;
    if (c == '{') {
      ++p_; j.kind = Json::Obj;
      if (peek() == '}') { ++p_; return j; }
      for (;;) {
        Json k = string();
        expect(':');
        j.o.emplace_back(k.s, value());
        if (peek() == ',') { ++p_; continue; }
        expect('}');
        return j;
      }
    }
    if (c == '[') {
      ++p_; j.kind = Json::Arr;
      if (peek() == ']') { ++p_; return j; }
      for (;;) {
        j.a.push_back(value());
        if (peek() == ',') { ++p_; continue; }
        expect(']');
        return j;
      }
    }
    if (c == '"') return string();
    if (!strncmp(p_, "true", 4) && e_ - p_ >= 4) { p_ += 4; j.kind = Json::Bool; j.b = true; return j; }
    if (!strncmp(p_, "false", 5) && e_ - p_ >= 5) { p_ += 5; j.kind = Json::Bool; j.b = false; return j; }
    if (!strncmp(p_, "null", 4) && e_ - p_ >= 4) { p_ += 4; return j; }
    const char* s = p_;
    while (p_ < e_ && (isdigit((unsigned char)*p_) || *p_ == '-' || *p_ == '+' || *p_ == '.' || *p_ == 'e' || *p_ == 'E')) ++p_;
    SG_CHECK(p_ > s, SAILGPU_ERR_INVALID, "spec: bad token");
    j.kind = Json::Num; j.s.assign(s, p_);
    return j;
  }
  Json string() {
    expect('"');
    Json j; j.kind = Json::Str;
    while (p_ < e_ && *p_ != '"') {
      if (*p_ == '\\' && p_ + 1 < e_) {
        ++p_;
        switch (*p_) {
          case 'n': j.s += '\n'; break; case 't': j.s += '\t'; break; case 'r': j.s += '\r'; break;
          case 'b': j.s += '\b'; break; case 'f': j.s += '\f'; break;
          case 'u': {
            SG_CHECK(e_ - p_ >= 5, SAILGPU_ERR_INVALID, "spec: bad \\u escape");
            unsigned cp = (unsigned)strtoul(std::string(p_ + 1, p_ + 5).c_str(), nullptr, 16);
            p_ += 4;
            if (cp < 0x80) j.s += (char)cp;
            else if (cp < 0x800) { j.s += (char)(0xC0 | (cp >> 6)); j.s += (char)(0x80 | (cp & 0x3F)); }
            else { j.s += (char)(0xE0 | (cp >> 12)); j.s += (char)(0x80 | ((cp >> 6) & 0x3F)); j.s += (char)(0x80 | (cp & 0x3F)); }
            break;
          }
          default: j.s += *p_;
        }
        ++p_;
      } else {
        j.s += *p_++;
      }
    }
    expect('"');
    return j;
  }
};

typedef __int128 i128;
typedef unsigned __int128 u128;

inline i128 parse_i128(const std::string& s) {
  bool neg = false; size_t i = 0;
  if (i < s.size() && (s[i] == '-' || s[i] == '+')) { neg = s[i] == '-'; ++i; }
  u128 v = 0;
  SG_CHECK(i < s.size(), SAILGPU_ERR_INVALID, "spec: empty integer literal");
  for (; i < s.size(); ++i) {
    SG_CHECK(isdigit((unsigned char)s[i]), SAILGPU_ERR_INVALID, "spec: bad integer literal '" + s + "'");
    v = v * 10 + (unsigned)(s[i] - '0');
  }
  return neg ? -(i128)v : (i128)v;
}
inline i128 pow10_i128(int k) { i128 v = 1; while (k-- > 0) v *= 10; return v; }

}  // namespace sg
