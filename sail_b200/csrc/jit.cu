// jit.cu -- pipeline specialiser (host side).
//
// The interpreter (pipeline.cu) runs any fused Filter -> Projection -> Aggregate chain at once; its cost is ~650 thread
// instructions per TPC-H Q1 row, most of them descriptor decoding and shared-memory round trips of intermediates.
// For pipelines that see enough rows this file writes the same pipeline as straight-line CUDA
// over registers -- one `struct G` per pipeline, consumed by the templates in jit_rt.cuh -- and compiles it with NVRTC
// for sm_90a.  No new operator semantics live here: every generated statement is the register form of one VM
// instruction (vm.h) or one sink descriptor.  Kernels are cached by source hash, in memory and as cubins next to the
// library (sail_b200/_build/jit_cache), so a pipeline is compiled once per machine.
#include "jit.hpp"

#include <dlfcn.h>
#include <sys/stat.h>
#include <unistd.h>

#include <chrono>
#include <fstream>
#include <mutex>
#include <sstream>
#include <tuple>

namespace sg {

// ================================================================================================
// source generation
// ================================================================================================
namespace {

const char* ctype(int k) {
  switch (k) {
    case K_B: return "bool";
    case K_I32: return "int32_t";
    case K_I64: return "int64_t";
    case K_F64: return "double";
    case K_I128: return "i128";
    default: return "ulonglong2";
  }
}
std::string hex64(uint64_t v) { char b[32]; snprintf(b, sizeof b, "0x%016llxull", (unsigned long long)v); return b; }
std::string lit(int kind, uint64_t i0, uint64_t i1) {
  char b[96];
  switch (kind) {
    case K_B: return (i0 & 1) ? "true" : "false";
    case K_I32: snprintf(b, sizeof b, "(int32_t)0x%08xu", (unsigned)(uint32_t)i0); return b;
    case K_I64: return "(int64_t)" + hex64(i0);
    case K_F64: return "__longlong_as_double((long long)" + hex64(i0) + ")";
    case K_I128: return "mk128(" + hex64(i0) + ", " + hex64(i1) + ")";
    default: return "mkv16(" + hex64(i0) + ", " + hex64(i1) + ")";
  }
}
uint32_t align128(uint32_t v) { return (v + 127) & ~127u; }

struct Unsupported { std::string why; };

struct Emitter {
  const CompiledPipeline& cp;
  const JitInfo& J;
  JitPlan plan;
  int tile;
  std::ostringstream body;                                   // statements of eval()
  std::map<int, int> input_index;                            // input slot id -> index in J.inputs
  std::vector<uint32_t> in_off, in_bytes;
  std::map<std::tuple<int, int, int>, std::string> loads;    // (slot, kind, stride) -> variable
  std::map<int, int> tkind;                                  // temp slot id -> kind
  std::vector<std::pair<std::string, std::string>> fields;   // Row fields (type, name)
  std::map<std::string, std::string> exported;               // variable -> Row field
  std::ostringstream exports;

  Emitter(const CompiledPipeline& c, const JitPlan& p) : cp(c), J(c.jit), plan(p), tile(p.rpt * NT) {
    uint32_t off = 0;
    for (size_t i = 0; i < J.inputs.size(); ++i) {
      const InputReg& r = J.inputs[i];
      input_index[r.slot] = (int)i;
      const uint32_t b = r.width ? (uint32_t)r.width * tile : (uint32_t)tile / 8;
      in_off.push_back(off); in_bytes.push_back(b);
      off += align128(b);
    }
  }
  bool is_input(int slot) const { return J.slots.at((size_t)slot).is_input; }

  static std::string load_expr(const char* type, const std::string& addr) {
    if (!strcmp(type, "ulonglong2")) return "*reinterpret_cast<const ulonglong2*>(" + addr + ")";
    if (!strcmp(type, "bool")) return "(*(" + addr + ") != 0)";
    return std::string("lds<") + type + ">(" + addr + ")";
  }
  // value of slot `slot` read as `kind`
  std::string operand(uint32_t slot_u, int kind, int stride) {
    if (slot_u == NO_SLOT) throw Unsupported{"operand without a slot"};
    const int slot = (int)slot_u;
    if (!is_input(slot)) {
      auto it = tkind.find(slot);
      if (it == tkind.end()) throw Unsupported{"temporary read before it is written"};
      if (it->second != kind) throw Unsupported{"temporary read with another kind"};
      return "t" + std::to_string(slot);
    }
    const InputReg& in = J.inputs[(size_t)input_index.at(slot)];
    if (in.width == 0) throw Unsupported{"bit-packed input read as a value"};
    if (stride <= 0) stride = in.width;
    auto key = std::make_tuple(slot, kind, stride);
    auto it = loads.find(key);
    if (it != loads.end()) return it->second;
    const std::string name = "i" + std::to_string(slot) + "_" + std::to_string(kind) + "_" + std::to_string(stride);
    body << "    const " << ctype(kind) << " " << name << " = "
         << load_expr(ctype(kind), "st + " + std::to_string(in_off[(size_t)input_index.at(slot)]) + " + r * " + std::to_string(stride)) << ";\n";
    loads[key] = name;
    return name;
  }
  // raw typed load of an input (OP_CVT sources: int8 ... float)
  std::map<std::tuple<int, std::string, int>, std::string> raw_loads;
  std::string raw_load(uint32_t slot_u, const char* type, int stride) {
    const int slot = (int)slot_u;
    auto key = std::make_tuple(slot, std::string(type), stride);
    auto it = raw_loads.find(key);
    if (it != raw_loads.end()) return it->second;
    const std::string name = "c" + std::to_string(slot) + "_" + std::to_string(raw_loads.size());
    body << "    const " << type << " " << name << " = "
         << load_expr(type, "st + " + std::to_string(in_off[(size_t)input_index.at(slot)]) + " + r * " + std::to_string(stride)) << ";\n";
    raw_loads[key] = name;
    return name;
  }
  void def(uint32_t dst, int kind, const std::string& expr) {
    body << "    const " << ctype(kind) << " t" << dst << " = " << expr << ";\n";
    tkind[(int)dst] = kind;
  }

  void emit_inst(int pc, const VmInst& I) {
    const int base = I.op & 0xFF, kind = I.op >> 8;
    const bool ia = I.flags & F_IMM_A, ib = I.flags & F_IMM_B;
    auto A = [&](int k) { return ia ? lit(k, I.imm0, I.imm1) : operand(I.a, k, I.sa); };
    auto B = [&](int k) { return ib ? lit(k, I.imm0, I.imm1) : operand(I.b, k, I.sb); };
    const std::string T = ctype(kind);
    switch (base) {
      case OP_NOP: break;
      case OP_UNPACK_BITS: {
        if (!is_input((int)I.a) || J.inputs[(size_t)input_index.at((int)I.a)].width != 0) throw Unsupported{"UNPACK_BITS of a non-bitmap slot"};
        const uint32_t off = in_off[(size_t)input_index.at((int)I.a)];
        def(I.dst, K_B, "((st[" + std::to_string(off) + " + (r >> 3)] >> (r & 7)) & 1) != 0");
        break;
      }
      case OP_CONST: def(I.dst, kind, lit(kind, I.imm0, I.imm1)); break;
      case OP_MOV: def(I.dst, kind, operand(I.a, kind, I.sa)); break;
      case OP_CVT: {
        static const char* src_t[] = {"int8_t", "int16_t", "uint8_t", "uint16_t", "uint32_t", "float", "int32_t", "int64_t", "double", "i128", "bool"};
        static const int src_k[] = {-1, -1, -1, -1, -1, -1, K_I32, K_I64, K_F64, K_I128, K_B};
        if (I.aux == SRC_U64) {   // UInt64 -> Float64, rounded once
          if (kind != K_F64) throw Unsupported{"CVT from UInt64 to an integer"};
          def(I.dst, kind, "(double)(uint64_t)" + operand(I.a, K_I64, I.sa)); break;
        }
        if (I.aux > SRC_B) throw Unsupported{"CVT source"};
        std::string x;
        if (is_input((int)I.a)) x = (src_k[I.aux] >= 0 && src_k[I.aux] != K_B) ? operand(I.a, src_k[I.aux], I.sa) : raw_load(I.a, src_t[I.aux], I.sa);
        else { if (src_k[I.aux] < 0) throw Unsupported{"narrow CVT of a temporary"}; x = operand(I.a, src_k[I.aux], I.sa); }
        def(I.dst, kind, "jit_cvt<" + T + ">(" + x + ")");
        break;
      }
      case OP_ADD: def(I.dst, kind, "OpAdd::f<" + T + ">(" + A(kind) + ", " + B(kind) + ")"); break;
      case OP_SUB: def(I.dst, kind, "OpSub::f<" + T + ">(" + A(kind) + ", " + B(kind) + ")"); break;
      case OP_MUL: def(I.dst, kind, "OpMul::f<" + T + ">(" + A(kind) + ", " + B(kind) + ")"); break;
      case OP_DIV: case OP_REM: {
        if (kind == K_F64) { def(I.dst, kind, base == OP_REM ? "fmod(" + A(kind) + ", " + B(kind) + ")" : A(kind) + " / " + B(kind)); break; }
        std::string live = "inb";
        if (I.c != NO_SLOT) live += " && " + operand(I.c, K_B, 1);
        def(I.dst, kind, "jit_div<" + T + ", " + (base == OP_REM ? "true" : "false") + ">(" + A(kind) + ", " + B(kind) + ", " + live + ", K.P[0].error_flag)");
        break;
      }
      case OP_NEG: {
        const std::string a = operand(I.a, kind, I.sa);
        if (kind == K_I32) def(I.dst, kind, "(int32_t)(0u - (uint32_t)" + a + ")");
        else if (kind == K_I64) def(I.dst, kind, "(int64_t)(0ull - (uint64_t)" + a + ")");
        else if (kind == K_F64) def(I.dst, kind, "-" + a);
        else def(I.dst, kind, "(i128)((u128)0 - (u128)" + a + ")");
        break;
      }
      case OP_MULW: def(I.dst, K_I128, "jit_mulw(" + A(K_I64) + ", " + B(K_I64) + ")"); break;
      case OP_MUL128_64: def(I.dst, K_I128, "jit_mul128_64(" + operand(I.a, K_I128, I.sa) + ", " + B(K_I64) + ")"); break;
      case OP_DIVROUND: def(I.dst, kind, "jit_divround<" + T + ">(" + operand(I.a, kind, I.sa) + ", " + lit(kind, I.imm0, I.imm1) + ")"); break;
      case OP_MUL_POW10_CHK: {
        const u128 p = ((u128)I.imm1 << 64) | I.imm0, lim = (~(u128)0 >> 1) / p;
        std::string live = "inb";
        if (I.c != NO_SLOT) live += " && " + operand(I.c, K_B, 1);
        def(I.dst, K_I128, "checked_mul_pow10(" + operand(I.a, K_I128, I.sa) + ", " + lit(K_I128, I.imm0, I.imm1) + ", " +
                               lit(K_I128, (uint64_t)lim, (uint64_t)(lim >> 64)) + ", " + live + ", K.P[0].error_flag)");
        break;
      }
      case OP_EQ: case OP_NE: case OP_LT: case OP_LE: case OP_GT: case OP_GE: {
        if (kind == K_V16) {
          if (base != OP_EQ && base != OP_NE) throw Unsupported{"ordering comparison of strings"};
          def(I.dst, K_B, std::string(base == OP_NE ? "!" : "") + "view_equal(" + A(K_V16) + ", " + B(K_V16) + ")");
        } else {
          static const char* ops[] = {"==", "!=", "<", "<=", ">", ">="};
          def(I.dst, K_B, "(" + A(kind) + " " + ops[base - OP_EQ] + " " + B(kind) + ")");
        }
        break;
      }
      case OP_AND: def(I.dst, K_B, "(" + A(K_B) + " && " + B(K_B) + ")"); break;
      case OP_OR: def(I.dst, K_B, "(" + A(K_B) + " || " + B(K_B) + ")"); break;
      case OP_ANDNOT: def(I.dst, K_B, "(" + A(K_B) + " && !" + B(K_B) + ")"); break;
      case OP_NOT: def(I.dst, K_B, "!" + A(K_B)); break;
      case OP_SELECT: def(I.dst, kind, "(" + operand(I.c, K_B, 1) + " ? " + A(kind) + " : " + B(kind) + ")"); break;
      case OP_STR_EQ_LONG:
        def(I.dst, K_B, std::string("((inb && view_equal(") + operand(I.a, K_V16, I.sa) + ", mkv16(" + hex64(I.imm0) + ", K.prog[0][" + std::to_string(pc) + "].imm1))) != " +
                            ((I.aux & 1) ? "true" : "false") + ")");
        break;
      case OP_STR_LIKE:
        def(I.dst, K_B, std::string("((inb && jit_like(") + operand(I.a, K_V16, I.sa) + ", reinterpret_cast<const uint8_t*>(K.prog[0][" + std::to_string(pc) + "].imm1), " +
                            std::to_string((uint32_t)I.imm0) + "u, " + std::to_string(I.aux & 0xFF) + ")) != " + (((I.aux >> 8) & 1) ? "true" : "false") + ")");
        break;
      case OP_SUBSTR:
        def(I.dst, K_V16, "(inb ? view_substr(" + operand(I.a, K_V16, I.sa) + ", " + std::to_string((long long)I.imm0) + "ll, " + std::to_string((long long)I.imm1) + "ll) : mkv16(0ull, 0ull))");
        break;
      case OP_CHAR_LEN: def(I.dst, K_I32, "(inb ? view_char_length(" + operand(I.a, K_V16, I.sa) + ") : 0)"); break;
      case OP_DATE_PART: def(I.dst, K_I32, "jit_date_part(" + operand(I.a, K_I32, I.sa) + ", " + std::to_string(I.aux) + ")"); break;
      case OP_TS_PART: case OP_TS_TRUNC: {   // unit and zone offset become constants: the divisions strength-reduce
        const std::string call = std::string(base == OP_TS_TRUNC ? "ts_trunc_u<" : "ts_part_u<") + std::to_string((long long)I.imm0) + "ll>(" +
                                 operand(I.a, K_I64, I.sa) + ", " + std::to_string(I.aux) + ", " + std::to_string((long long)I.imm1) + "ll)";
        def(I.dst, kind, kind == K_I32 ? "(int32_t)" + call : call);
        break;
      }
      default: throw Unsupported{"VM instruction " + std::to_string(base)};
    }
  }

  // Row field carrying slot `slot` (read as `kind`) out of eval()
  std::string field(uint32_t slot, int kind, int stride) {
    const std::string var = operand(slot, kind, stride);
    auto it = exported.find(var);
    if (it != exported.end()) return it->second;
    const std::string f = "f" + std::to_string(fields.size());
    fields.emplace_back(ctype(kind), f);
    exports << "    o." << f << " = " << var << ";\n";
    exported[var] = f;
    return f;
  }
  int value_kind(uint32_t slot, int width, bool is_view) {
    if (!is_input((int)slot)) { auto it = tkind.find((int)slot); if (it == tkind.end()) throw Unsupported{"sink reads an undefined slot"}; return it->second; }
    return width == 16 ? (is_view ? K_V16 : K_V16) : width == 8 ? K_I64 : width == 4 ? K_I32 : K_B;
  }
  static std::string chain(const std::vector<int>& v) {     // j == 0 ? v0 : j == 1 ? v1 : ... : 0
    std::string s;
    for (size_t j = 0; j < v.size(); ++j) s += "j == " + std::to_string(j) + " ? " + std::to_string(v[j]) + " : ";
    return s + "0";
  }

  std::string gen_agg() {
    const AggParams& A = J.agg;
    std::ostringstream o;
    const int tier = A.cold_only ? 0 : A.reg_path ? 2 : A.hot_groups > 0 ? 1 : 0;
    const int hot_g = std::min(HOT_MAX_GROUPS, std::max(A.hot_groups, tier == 2 ? REG_GROUPS : 0));
    std::vector<int> ops, words, seen, modes;
    for (int j = 0; j < A.n_accs; ++j) {
      ops.push_back(A.accs[j].op); words.push_back(A.accs[j].word); seen.push_back(A.accs[j].track_seen);
      modes.push_back(A.accs[j].op == ACC_COUNT ? 0 : A.accs[j].vkind == K_I64 ? (J.small_acc[j] ? 3 : 1) : 2);
    }
    // the key in registers is padded to the dictionary's HOT_KEY_WORDS words (those tiers compare and fingerprint four words)
    const int key_regs = std::max(A.key_words, HOT_KEY_WORDS);
    o << "  static constexpr int N_KEYS = " << A.n_keys << ", KEY_WORDS = " << A.key_words << ", N_ACCS = " << A.n_accs << ", ENTRY_WORDS = " << (2 + A.key_words + A.acc_words)
      << ", HOT_G = " << std::max(hot_g, 1) << ", AGG_TIER = " << tier << ";\n";
    o << "  using Key = JitKey<" << key_regs << ">;\n";
    o << "  static __device__ __forceinline__ constexpr int acc_op(int j) { return " << chain(ops) << "; }\n";
    o << "  static __device__ __forceinline__ constexpr int acc_word(int j) { return " << chain(words) << "; }\n";
    o << "  static __device__ __forceinline__ constexpr int acc_seen(int j) { return " << chain(seen) << "; }\n";
    o << "  static __device__ __forceinline__ constexpr int reg_mode(int j) { return " << chain(modes) << "; }\n";
    // key words
    std::ostringstream kwf, khf, kef;
    kwf << "  static __device__ __forceinline__ void key_words(const Row& o, Key& k) {\n";
    khf << "  static __device__ __forceinline__ uint64_t key_hash(const Key& k) {\n    uint64_t h = 0x243F6A8885A308D3ull;\n";
    kef << "  static __device__ __forceinline__ bool keys_equal(const uint64_t* a, const Key& k) {\n    bool eq = true;\n";
    if (A.has_null_word) { kwf << "    uint64_t nm = 0;\n"; kef << "    eq = eq && a[0] == k.w[0];\n"; }
    int w = A.has_null_word ? 1 : 0;
    for (int i = 0; i < A.n_keys; ++i) {
      const KeyDesc& k = A.keys[i];
      const int kk = value_kind(k.slot, k.width, k.is_view != 0);
      const std::string f = "o." + field(k.slot, kk, k.stride);
      std::string nul = "false";
      if (k.valid_slot != NO_SLOT) { nul = "!o." + field(k.valid_slot, K_B, 1); kwf << "    if (" << nul << ") nm |= " << (1ull << i) << "ull;\n"; }
      if (k.width == 16) {
        if (kk == K_V16) kwf << "    k.w[" << w << "] = " << nul << " ? 0ull : " << f << ".x; k.w[" << w + 1 << "] = " << nul << " ? 0ull : " << f << ".y;\n";
        else kwf << "    k.w[" << w << "] = " << nul << " ? 0ull : i128_lo(" << f << "); k.w[" << w + 1 << "] = " << nul << " ? 0ull : i128_hi(" << f << ");\n";
        const std::string v = "mkv16(k.w[" + std::to_string(w) + "], k.w[" + std::to_string(w + 1) + "])";
        if (k.is_view) {
          khf << "    h = mix64(h ^ view_hash(" << v << "));\n";
          kef << "    eq = eq && view_equal(mkv16(a[" << w << "], a[" << w + 1 << "]), " << v << ");\n";
        } else {
          khf << "    h = mix64(h ^ mix64(k.w[" << w << "] ^ mix64(k.w[" << w + 1 << "])));\n";
          kef << "    eq = eq && a[" << w << "] == k.w[" << w << "] && a[" << w + 1 << "] == k.w[" << w + 1 << "];\n";
        }
        w += 2;
      } else {
        std::string bits;
        if (kk == K_I64) bits = "(uint64_t)" + f;
        else if (kk == K_F64) bits = "(uint64_t)__double_as_longlong(" + f + ")";
        else if (kk == K_I32) bits = "(uint64_t)(uint32_t)" + f;
        else if (kk == K_B) bits = "(" + f + " ? 1ull : 0ull)";
        else throw Unsupported{"group key kind"};
        kwf << "    k.w[" << w << "] = " << nul << " ? 0ull : " << bits << ";\n";
        khf << "    h = mix64(h ^ k.w[" << w << "]);\n";
        kef << "    eq = eq && a[" << w << "] == k.w[" << w << "];\n";
        w += 1;
      }
    }
    if (A.has_null_word) { kwf << "    k.w[0] = nm;\n"; khf << "    h = mix64(h ^ k.w[0]);\n"; }
    for (int z = w; z < key_regs; ++z) kwf << "    k.w[" << z << "] = 0ull;\n";
    kwf << "  }\n"; khf << "    return h;\n  }\n"; kef << "    return eq;\n  }\n";
    o << kwf.str() << khf.str() << kef.str();
    // accumulator inputs
    o << "  template <int J> static __device__ __forceinline__ AccVal acc(const Row& o) {\n    AccVal v; v.i = 0; v.f = 0.0; v.valid = true;\n";
    for (int j = 0; j < A.n_accs; ++j) {
      const AccDesc& d = A.accs[j];
      o << "    if constexpr (J == " << j << ") {";
      if (d.valid_slot != NO_SLOT) o << " v.valid = o." << field(d.valid_slot, K_B, 1) << ";";
      if (d.value_slot != NO_SLOT) {
        const std::string f = "o." + field(d.value_slot, d.vkind, d.stride);
        if (d.vkind == K_F64) o << " v.f = " << f << ";";
        else if (d.vkind == K_B) o << " v.i = " << f << " ? 1 : 0;";
        else if (d.vkind == K_V16) throw Unsupported{"string accumulator"};
        else o << " v.i = (i128)" << f << ";";
      }
      if (acc_is_dd(d.op)) {   // the double-double term (pipeline.cu set_dd_value): high part in f, low part in i
        if (d.vkind != K_F64) throw Unsupported{"variance accumulator over a non-Float64 slot"};
        const bool merging = d.n_slot != NO_SLOT;
        const std::string n = merging ? "o." + field(d.n_slot, K_F64, 8) : "0.0", mean = merging ? "o." + field(d.mean_slot, K_F64, 8) : "0.0";
        o << " { double h, l; dd_term(" << (int)d.op << ", v.f, " << n << ", " << mean << ", " << (merging ? "true" : "false")
          << ", h, l); v.f = h; v.i = (i128)(uint64_t)__double_as_longlong(l); }";
      }
      o << " }\n";
    }
    o << "    return v;\n  }\n";
    return o.str();
  }

  std::string gen_outputs() {
    std::ostringstream o;
    std::vector<int> widths, nullable;
    for (auto& c : J.outs) { widths.push_back(c.width); nullable.push_back(c.valid_slot != NO_SLOT ? 1 : 0); }
    o << "  static constexpr int N_OUT = " << J.outs.size() << ";\n";
    o << "  static __device__ __forceinline__ constexpr int out_width(int j) { return " << chain(widths) << "; }\n";
    o << "  static __device__ __forceinline__ constexpr int out_nullable(int j) { return " << chain(nullable) << "; }\n";
    std::ostringstream st, ob, ov;
    st << "  template <int J> static __device__ __forceinline__ void store(const Row& o, uint8_t* data, int64_t pos) {\n";
    ob << "  template <int J> static __device__ __forceinline__ bool out_bool(const Row& o) {\n";
    ov << "  template <int J> static __device__ __forceinline__ bool out_valid(const Row& o) {\n";
    for (size_t j = 0; j < J.outs.size(); ++j) {
      const OutputCol& c = J.outs[j];
      int kind = J.out_kinds.at(j);
      if (c.width == 0) { ob << "    if constexpr (J == " << j << ") return o." << field(c.slot, K_B, 1) << ";\n"; }
      else {
        // an input column passed through keeps its raw bytes (a narrow decimal read as its low word is still 16 bytes wide)
        if (is_input((int)c.slot) && c.width == 16) kind = K_V16;
        const std::string f = "o." + field(c.slot, kind, c.stride);
        st << "    if constexpr (J == " << j << ") { ";
        if (c.width == 16) {
          if (kind == K_V16) st << "*reinterpret_cast<ulonglong2*>(data + pos * 16) = " << f << ";";
          else if (kind == K_I128) st << "*reinterpret_cast<ulonglong2*>(data + pos * 16) = mkv16(i128_lo(" << f << "), i128_hi(" << f << "));";
          else if (kind == K_I64) st << "*reinterpret_cast<ulonglong2*>(data + pos * 16) = mkv16((uint64_t)" << f << ", (uint64_t)(" << f << " >> 63));";
          else throw Unsupported{"16-byte output of kind " + std::to_string(kind)};
        } else if (c.width == 8) {
          if (kind == K_F64) st << "*reinterpret_cast<double*>(data + pos * 8) = " << f << ";";
          else if (kind == K_I64) st << "*reinterpret_cast<int64_t*>(data + pos * 8) = " << f << ";";
          else throw Unsupported{"8-byte output of kind " + std::to_string(kind)};
        } else if (c.width == 4 && kind == K_I32) st << "*reinterpret_cast<int32_t*>(data + pos * 4) = " << f << ";";
        else if (c.width == 2 && kind == K_I32) st << "*reinterpret_cast<uint16_t*>(data + pos * 2) = (uint16_t)(uint32_t)" << f << ";";
        else if (c.width == 1 && kind == K_I32) st << "data[pos] = (uint8_t)(uint32_t)" << f << ";";
        else throw Unsupported{"output width " + std::to_string(c.width) + " of kind " + std::to_string(kind)};
        st << " }\n";
      }
      if (c.valid_slot != NO_SLOT) ov << "    if constexpr (J == " << j << ") return o." << field(c.valid_slot, K_B, 1) << ";\n";
    }
    st << "  }\n"; ob << "    return false;\n  }\n"; ov << "    return true;\n  }\n";
    o << st.str() << ob.str() << ov.str();
    return o.str();
  }

  std::string run() {
    for (size_t pc = 0; pc < J.prog.size(); ++pc) emit_inst((int)pc, J.prog[pc]);
    std::string sink;
    if (cp.sink == SINK_AGG) sink = gen_agg();
    else sink = "  static constexpr int N_ACCS = 0, AGG_TIER = -1;\n" + gen_outputs();
    std::string live = "inb";
    if (J.mask.is_imm) { if (!(J.mask.i0 & 1)) throw Unsupported{"constant FALSE predicate"}; }
    else if (J.mask.slot >= 0) live += " && " + operand((uint32_t)J.mask.slot, K_B, 1);
    uint32_t stage_bytes = 0, tx = 0;
    for (size_t i = 0; i < in_bytes.size(); ++i) { stage_bytes = in_off[i] + align128(in_bytes[i]); tx += in_bytes[i]; }
    std::ostringstream o;
    o << "#include \"jit_rt.cuh\"\nnamespace sg {\nstruct G {\n";
    o << "  static constexpr int RPT = " << plan.rpt << ", STAGES = " << plan.stages << ", TILE = " << tile << ", SINK = " << cp.sink << ", N_IN = " << J.inputs.size() << ";\n";
    o << "  static constexpr uint32_t STAGE_BYTES = " << stage_bytes << "u, SCRATCH_BYTES = " << plan.scratch_bytes << "u, TX_BYTES = " << tx << "u;\n";
    o << "  struct Row {\n    bool live;\n";
    for (auto& f : fields) o << "    " << f.first << " " << f.second << ";\n";
    o << "  };\n";
    o << "  static __device__ __forceinline__ void issue(uint8_t* st, const KernelArgs& K, int64_t row0, uint64_t* bar) {\n";
    for (size_t i = 0; i < J.inputs.size(); ++i) {
      const InputReg& r = J.inputs[i];
      o << "    tma_load_1d(st + " << in_off[i] << ", K.P[0].in[" << i << "].data + " << (r.width ? "row0 * " + std::to_string(r.width) : std::string("(row0 >> 3)")) << ", " << in_bytes[i] << "u, bar);\n";
    }
    o << "  }\n";
    o << "  static __device__ __forceinline__ void copy_partial(uint8_t* st, const KernelArgs& K, int64_t row0, int nrows) {\n";
    for (size_t i = 0; i < J.inputs.size(); ++i) {
      const InputReg& r = J.inputs[i];
      o << "    jit_copy_col(st + " << in_off[i] << ", K.P[0].in[" << i << "].data + " << (r.width ? "row0 * " + std::to_string(r.width) : std::string("(row0 >> 3)")) << ", " << in_bytes[i] << "u, "
        << (r.width ? "(uint32_t)nrows * " + std::to_string(r.width) + "u" : std::string("(uint32_t)((nrows + 7) >> 3)")) << ", K.P[0].in[" << i << "].tma_ok != 0);\n";
    }
    o << "  }\n";
    o << "  static __device__ __forceinline__ void eval(const uint8_t* st, int r, bool inb, const KernelArgs& K, Row& o) {\n";
    o << body.str() << exports.str() << "    o.live = " << live << ";\n  }\n";
    o << sink;
    o << "};\n}  // namespace sg\n";
    o << "extern \"C\" __global__ void __launch_bounds__(" << NT << ", " << plan.minb << ") sg_jit_kernel(const __grid_constant__ sg::KernelArgs K) { sg::jit_main<sg::G>(K); }\n";
    return o.str();
  }
};

int env_i(const char* n, int d) { const char* v = getenv(n); return v && *v ? atoi(v) : d; }

}  // namespace

bool jit_enabled() { return env_i("SAILGPU_JIT", 1) != 0; }      // read per launch: a host can turn specialisation off at run time
int64_t jit_min_rows() { const char* v = getenv("SAILGPU_JIT_MIN_ROWS"); return v && *v ? atoll(v) : (int64_t)4 << 20; }

bool jit_supported(const CompiledPipeline& cp, std::string* why) {
  auto no = [&](const char* w) { if (why) *why = w; return false; };
  if (!cp.jit.valid) return no("no specialiser snapshot");
  if (cp.sink != SINK_AGG && cp.sink != SINK_STORE && cp.sink != SINK_COMPACT) return no("sink is not aggregate / store / compact");
  if (cp.jit.inputs.empty()) return no("pipeline reads no column");
  // a specialised probe that resolves one row at a time was slower on orders x lineitem when it was measured (not on H100):
  // the interpreter issues the first-slot loads of all rows of a thread before the dependent key loads, and latency, not
  // instructions, bounds a probe
  if (cp.n_probes > 0) return no("join probes run on the interpreter");
  // the gate of a DISTINCT aggregate (a pair-set lookup per row) is not generated yet
  if (!cp.distinct.empty()) return no("DISTINCT aggregates (OP_DISTINCT_FIRST gates) run on the interpreter");
  return true;
}

bool jit_plan(const CompiledPipeline& cp, size_t max_smem, JitPlan* plan) {
  const JitInfo& J = cp.jit;
  JitPlan p;
  p.rpt = cp.rpt;
  const uint32_t tile = (uint32_t)p.rpt * NT;
  uint32_t stage = 0;
  for (auto& r : J.inputs) stage += align128(r.width ? (uint32_t)r.width * tile : tile / 8);
  p.stage_bytes = stage;
  int target = 3, cap = p.rpt >= 4 ? 2 : 3, max_s = 4;
  if (cp.sink == SINK_AGG) {
    const AggParams& A = J.agg;
    const int tier = A.cold_only ? 0 : A.reg_path ? 2 : A.hot_groups > 0 ? 1 : 0;
    const int hot_g = std::min(HOT_MAX_GROUPS, std::max(A.hot_groups, tier == 2 ? REG_GROUPS : 0));
    if (tier > 0) p.scratch_bytes = hot_scratch_bytes(hot_g, A.n_accs);
    target = tier == 0 ? 3 : 2; cap = tier == 0 ? 4 : 2;
    // dictionary / register tiers: two stages streamed faster than three or four on H100 (DESIGN.md section 4.1)
    if (tier > 0) max_s = 2;
  }
  const int force_s = env_i("SAILGPU_JIT_STAGES", 0);
  int chosen = 0;
  for (int s = 4; s >= 2 && !chosen; --s) {
    if (force_s ? s != force_s : s > max_s) continue;
    const size_t smem = JIT_HDR_BYTES + p.scratch_bytes + (size_t)s * stage;
    if (smem > max_smem) continue;
    const int ctas = (int)((228 * 1024) / (smem + 1024));
    if (ctas >= target || force_s) chosen = s;
  }
  if (!chosen) {
    const size_t smem = JIT_HDR_BYTES + p.scratch_bytes + 2 * (size_t)stage;
    if (smem > max_smem) return false;
    chosen = 2;
  }
  p.stages = chosen;
  p.smem_bytes = JIT_HDR_BYTES + p.scratch_bytes + (size_t)chosen * stage;
  const int by_smem = std::max(1, (int)((228 * 1024) / (p.smem_bytes + 1024)));
  p.minb = std::max(1, std::min(by_smem, env_i("SAILGPU_JIT_MINB", cap)));
  *plan = p;
  return true;
}

std::string jit_generate(const CompiledPipeline& cp, const JitPlan& plan) {
  try {
    Emitter e(cp, plan);
    return e.run();
  } catch (const Unsupported& u) {
    fail(SAILGPU_ERR_UNSUPPORTED, "kernel specialiser: " + u.why);
  }
}

// ================================================================================================
// NVRTC + driver API (both dlopen'ed: the library loads without them; a pipeline then stays on the interpreter)
// ================================================================================================
namespace {

// headers of the generated translation unit, embedded at build time (sail_b200/build.py -> _build/jit_headers.inc)
struct EmbeddedHeader { const char* name; const char* text; };
#include "../_build/jit_headers.inc"

const char* kStdint =
    "#pragma once\n"
    "typedef signed char int8_t; typedef short int16_t; typedef int int32_t; typedef long long int64_t;\n"
    "typedef unsigned char uint8_t; typedef unsigned short uint16_t; typedef unsigned int uint32_t; typedef unsigned long long uint64_t;\n";

struct Nvrtc {
  void* h = nullptr;
  int (*CreateProgram)(void**, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
  int (*CompileProgram)(void*, int, const char* const*) = nullptr;
  int (*GetCUBINSize)(void*, size_t*) = nullptr;
  int (*GetCUBIN)(void*, char*) = nullptr;
  int (*GetProgramLogSize)(void*, size_t*) = nullptr;
  int (*GetProgramLog)(void*, char*) = nullptr;
  int (*DestroyProgram)(void**) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  std::string err;
};
Nvrtc& nvrtc() {
  static Nvrtc n;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so"};
    for (const char* nm : names) { n.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (n.h) break; }
    if (!n.h) { n.err = "libnvrtc.so.12 not found"; return; }
#define SG_SYM(field, sym) *(void**)(&n.field) = dlsym(n.h, sym); if (!n.field) { n.err = std::string("missing symbol ") + sym; return; }
    SG_SYM(CreateProgram, "nvrtcCreateProgram") SG_SYM(CompileProgram, "nvrtcCompileProgram") SG_SYM(GetCUBINSize, "nvrtcGetCUBINSize")
    SG_SYM(GetCUBIN, "nvrtcGetCUBIN") SG_SYM(GetProgramLogSize, "nvrtcGetProgramLogSize") SG_SYM(GetProgramLog, "nvrtcGetProgramLog")
    SG_SYM(DestroyProgram, "nvrtcDestroyProgram") SG_SYM(GetErrorString, "nvrtcGetErrorString")
#undef SG_SYM
  });
  return n;
}

struct Driver {
  void* h = nullptr;
  int (*ModuleLoadData)(void**, const void*) = nullptr;
  int (*ModuleGetFunction)(void**, void*, const char*) = nullptr;
  int (*FuncSetAttribute)(void*, int, int) = nullptr;
  int (*OccupancyMaxActiveBlocksPerMultiprocessor)(int*, void*, int, size_t) = nullptr;
  int (*LaunchKernel)(void*, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, void*, void**, void**) = nullptr;
  int (*GetErrorString)(int, const char**) = nullptr;
  std::string err;
};
Driver& driver() {
  static Driver d;
  static std::once_flag once;
  std::call_once(once, [] {
    d.h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!d.h) { d.err = "libcuda.so.1 not found"; return; }
#define SG_SYM(field, sym) *(void**)(&d.field) = dlsym(d.h, sym); if (!d.field) { d.err = std::string("missing symbol ") + sym; return; }
    SG_SYM(ModuleLoadData, "cuModuleLoadData") SG_SYM(ModuleGetFunction, "cuModuleGetFunction") SG_SYM(FuncSetAttribute, "cuFuncSetAttribute")
    SG_SYM(OccupancyMaxActiveBlocksPerMultiprocessor, "cuOccupancyMaxActiveBlocksPerMultiprocessor") SG_SYM(LaunchKernel, "cuLaunchKernel")
    SG_SYM(GetErrorString, "cuGetErrorString")
#undef SG_SYM
  });
  return d;
}
std::string cu_err(int e) { const char* s = nullptr; if (driver().GetErrorString) driver().GetErrorString(e, &s); return s ? s : ("CUresult " + std::to_string(e)); }

uint64_t fnv1a(const std::string& s, uint64_t seed) {
  uint64_t h = 0xcbf29ce484222325ull ^ seed;
  for (unsigned char c : s) { h ^= c; h *= 0x100000001b3ull; }
  return h;
}
static const char kJitArch[] = "sm_90a";
std::string runtime_fingerprint() {       // the target architecture and the embedded headers are part of every kernel's identity
  static const std::string fp = [] {
    std::string all = kJitArch;
    for (const EmbeddedHeader* h = kJitHeaders; h->name; ++h) { all += h->name; all += h->text; }
    char b[40]; snprintf(b, sizeof b, "%016llx", (unsigned long long)fnv1a(all, 17));
    return std::string(b);
  }();
  return fp;
}
std::string cache_dir() {
  static const std::string dir = [] {
    const char* e = getenv("SAILGPU_JIT_CACHE");
    std::string d;
    if (e && *e) d = e;
    else {
      Dl_info info;
      if (dladdr((void*)&cache_dir, &info) && info.dli_fname) { d = info.dli_fname; const size_t p = d.rfind('/'); d = (p == std::string::npos ? std::string(".") : d.substr(0, p)) + "/jit_cache"; }
      else d = "/tmp/sailgpu_jit_cache";
    }
    mkdir(d.c_str(), 0755);
    return d;
  }();
  return dir;
}

std::mutex g_jit_mu;
std::map<std::string, std::shared_ptr<JitKernel>> g_kernels;     // by source key

}  // namespace

std::string jit_compile_cubin(const std::string& source) {
  Nvrtc& n = nvrtc();
  SG_CHECK(n.err.empty(), SAILGPU_ERR_UNSUPPORTED, "NVRTC unavailable: " + n.err);
  std::vector<const char*> names, texts;
  for (const EmbeddedHeader* h = kJitHeaders; h->name; ++h) { names.push_back(h->name); texts.push_back(h->text); }
  names.push_back("stdint.h"); texts.push_back(kStdint);
  names.push_back("cuda_runtime.h"); texts.push_back("#pragma once\n");
  void* prog = nullptr;
  int rc = n.CreateProgram(&prog, source.c_str(), "sg_jit_kernel.cu", (int)names.size(), texts.data(), names.data());
  SG_CHECK(rc == 0, SAILGPU_ERR_CUDA, std::string("nvrtcCreateProgram: ") + n.GetErrorString(rc));
  const std::string arch = std::string("--gpu-architecture=") + kJitArch;
  const char* opts[] = {arch.c_str(), "--std=c++17", "-lineinfo", "-default-device", "--device-int128"};
  rc = n.CompileProgram(prog, 5, opts);
  if (rc != 0) {
    size_t ls = 0; n.GetProgramLogSize(prog, &ls);
    std::string log(ls, '\0');
    if (ls) n.GetProgramLog(prog, &log[0]);
    n.DestroyProgram(&prog);
    if (getenv("SAILGPU_JIT_DUMP")) fprintf(stderr, "%s\n", source.c_str());
    fail(SAILGPU_ERR_CUDA, std::string("NVRTC: ") + n.GetErrorString(rc) + "\n" + log.substr(0, 4000));
  }
  size_t sz = 0;
  rc = n.GetCUBINSize(prog, &sz);
  std::string cubin(sz, '\0');
  if (rc == 0 && sz) rc = n.GetCUBIN(prog, &cubin[0]);
  n.DestroyProgram(&prog);
  SG_CHECK(rc == 0 && sz > 0, SAILGPU_ERR_CUDA, "NVRTC produced no cubin");
  return cubin;
}

static std::string kernel_key(const std::string& source) {
  char b[64];
  snprintf(b, sizeof b, "%016llx%016llx", (unsigned long long)fnv1a(source, 1), (unsigned long long)fnv1a(source, 0x9E3779B97F4A7C15ull));
  return runtime_fingerprint() + "_" + b;
}

static void write_cache_file(const std::string& path, const std::string& cubin) {
  const std::string tmp = path + ".tmp" + std::to_string((long)getpid());
  std::ofstream f(tmp, std::ios::binary);
  if (f) { f.write(cubin.data(), (std::streamsize)cubin.size()); f.close(); rename(tmp.c_str(), path.c_str()); }
}

size_t jit_precompile_to_cache(const std::string& source) {
  const std::string path = cache_dir() + "/" + kernel_key(source) + ".cubin";
  struct stat st;
  if (stat(path.c_str(), &st) == 0 && st.st_size > 0) return (size_t)st.st_size;
  const std::string cubin = jit_compile_cubin(source);
  write_cache_file(path, cubin);
  return cubin.size();
}

bool jit_cached(const CompiledPipeline& cp, size_t max_smem) {
  std::string why;
  if (!jit_supported(cp, &why)) return false;
  JitPlan plan;
  if (!jit_plan(cp, max_smem, &plan)) return false;
  std::string src;
  try { src = jit_generate(cp, plan); } catch (const Error&) { return false; }
  const std::string key = kernel_key(src);
  {
    std::lock_guard<std::mutex> g(g_jit_mu);
    if (g_kernels.count(key)) return true;
  }
  return access((cache_dir() + "/" + key + ".cubin").c_str(), R_OK) == 0;
}

std::shared_ptr<JitKernel> jit_get_kernel(const CompiledPipeline& cp, size_t max_smem) {
  std::string why;
  SG_CHECK(jit_supported(cp, &why), SAILGPU_ERR_UNSUPPORTED, "kernel specialiser: " + why);
  JitPlan plan;
  SG_CHECK(jit_plan(cp, max_smem, &plan), SAILGPU_ERR_UNSUPPORTED, "kernel specialiser: pipeline does not fit in shared memory");
  const std::string src = jit_generate(cp, plan);
  if (getenv("SAILGPU_JIT_DUMP")) fprintf(stderr, "[sailgpu jit] source:\n%s\n", src.c_str());
  const std::string key = kernel_key(src);
  std::lock_guard<std::mutex> g(g_jit_mu);
  auto it = g_kernels.find(key);
  if (it != g_kernels.end()) return it->second;
  Driver& d = driver();
  SG_CHECK(d.err.empty(), SAILGPU_ERR_UNSUPPORTED, "CUDA driver API unavailable: " + d.err);
  std::string cubin;
  const std::string path = cache_dir() + "/" + key + ".cubin";
  {
    std::ifstream f(path, std::ios::binary);
    if (f) { std::stringstream ss; ss << f.rdbuf(); cubin = ss.str(); }
  }
  if (cubin.empty()) {
    const auto t0 = std::chrono::steady_clock::now();
    cubin = jit_compile_cubin(src);
    if (getenv("SAILGPU_JIT_VERBOSE"))
      fprintf(stderr, "[sailgpu jit] compiled %s in %.0f ms (%zu B)\n", key.c_str(),
              std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(), cubin.size());
    write_cache_file(path, cubin);
  }
  cudaFree(0);      // make sure the runtime's primary context is current on this thread
  auto k = std::make_shared<JitKernel>();
  int rc = d.ModuleLoadData(&k->module, cubin.data());
  SG_CHECK(rc == 0, SAILGPU_ERR_CUDA, "cuModuleLoadData: " + cu_err(rc));
  rc = d.ModuleGetFunction(&k->func, k->module, "sg_jit_kernel");
  SG_CHECK(rc == 0, SAILGPU_ERR_CUDA, "cuModuleGetFunction: " + cu_err(rc));
  rc = d.FuncSetAttribute(k->func, 8 /* CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES */, (int)plan.smem_bytes);
  SG_CHECK(rc == 0, SAILGPU_ERR_CUDA, "cuFuncSetAttribute: " + cu_err(rc));
  int per_sm = 0;
  rc = d.OccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k->func, NT, plan.smem_bytes);
  SG_CHECK(rc == 0 && per_sm >= 1, SAILGPU_ERR_CUDA, "specialised kernel cannot be resident: " + cu_err(rc));
  k->rpt = plan.rpt; k->stages = plan.stages; k->minb = plan.minb; k->smem_bytes = plan.smem_bytes; k->ctas_per_sm = per_sm; k->key = key;
  g_kernels[key] = k;
  return k;
}

void jit_launch(const JitKernel& k, const KernelArgs& K, int grid, cudaStream_t stream) {
  Driver& d = driver();
  void* params[] = {const_cast<KernelArgs*>(&K)};
  const int rc = d.LaunchKernel(k.func, (unsigned)grid, 1, 1, NT, 1, 1, (unsigned)k.smem_bytes, stream, params, nullptr);
  SG_CHECK(rc == 0, SAILGPU_ERR_CUDA, "cuLaunchKernel: " + cu_err(rc));
}

}  // namespace sg
