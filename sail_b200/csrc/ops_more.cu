// ops_more.cu -- HashJoinExec, SortExec / TopK, hash RepartitionExec and the NCCL all-to-all exchange.
//
// Reference call sites these replace (lakehq/sail):
//   HashJoinExec::try_new        crates/sail-execution/src/job_graph/planner.rs:137-147 (build = LEFT child,
//                                CollectLeft: crates/sail-physical-optimizer/src/collect_left.rs:40-53)
//   SortExec / TopK              crates/sail-session/src/planner.rs:7,34 ; plans test_tpch.plan.yaml:10,27,79
//   RepartitionExec Hash / BatchPartitioner + shuffle_write / shuffle_read
//                                crates/sail-execution/src/plan/shuffle_write.rs:173-196,209-267 ; shuffle_read.rs:107-117
#include <dlfcn.h>

#include "relational.hpp"
#include "runner.hpp"

namespace sg {

// ================================================================================================
// HashJoinExec
// ================================================================================================
struct JoinOp : Op {
  std::string jt;
  std::vector<int> lkeys, rkeys;
  Json filter_json; bool has_filter = false;
  std::vector<int> projection; bool has_proj = false;
  Schema bs, ps, joined;            // joined = what projection indexes (side schema for semi/anti)
  std::vector<BatchPtr> bparts;
  BatchPtr build;
  bool build_done = false, probe_done = false, tail_done = false;
  BufPtr table, dupflag, visited, next;
  uint64_t capacity = 0;
  bool dup = false;
  std::vector<BufPtr> build_valid_bytes, build_bool_bytes;
  std::vector<BufPtr> build_heaps;
  PipelineRunner brun, prun, frun, trun;
  ProbeParams pp{};
  std::map<const CompiledPipeline*, ProbeParams> pps;   // per compiled variant (validity signature)
  std::deque<BatchPtr> pending, ready;

  bool probe_streams_output() const { return jt == "inner" || jt == "right" || jt == "left" || jt == "right_semi" || jt == "right_anti"; }
  bool needs_visited() const { return jt == "left" || jt == "left_semi" || jt == "left_anti"; }
  bool general_path() const { return dup && (jt == "inner" || jt == "left" || jt == "right"); }

  void push(int input, const BatchPtr& b) override {
    const uint64_t t0 = now_ns();
    if (input == 0) {
      SG_CHECK(!build_done, SAILGPU_ERR_STATE, "build input already finished");
      bparts.push_back(b);
      m.build_input_rows += (uint64_t)b->rows; m.build_input_batches++;
      m.build_time_ns += now_ns() - t0;
      return;
    }
    SG_CHECK(input == 1, SAILGPU_ERR_INVALID, "hash_join has two inputs");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    if (!build_done) { pending.push_back(b); return; }
    probe(b);
    m.join_time_ns += now_ns() - t0;
    m.elapsed_compute_ns += now_ns() - t0;
  }
  void finish(int input) override {
    const uint64_t t0 = now_ns();
    if (input == 0) {
      finish_build();
      m.build_time_ns += now_ns() - t0;
      while (!pending.empty()) { probe(pending.front()); pending.pop_front(); }
      if (probe_done) emit_tail();
    } else {
      probe_done = true;
      if (build_done) emit_tail();
    }
    m.elapsed_compute_ns += now_ns() - t0;
  }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (!ready.empty()) {
      *out = ready.front(); ready.pop_front();
      m.output_rows += (uint64_t)(*out)->rows; m.output_batches++;
      return !(tail_done && ready.empty());
    }
    return !tail_done;
  }

  // ---- build -----------------------------------------------------------------------------------
  void finish_build() {
    build = concat_batches(ctx, bs, bparts);
    bparts.clear();
    build_done = true;
    const int64_t n = build->rows;
    capacity = next_pow2(std::max<uint64_t>(16, 2 * (uint64_t)n));
    table = dev_alloc_zero(ctx, (size_t)capacity * 16);
    dupflag = dev_alloc_zero(ctx, 16);
    next = dev_alloc(ctx, (size_t)n * 8 + 16);
    if (needs_visited()) visited = dev_alloc_zero(ctx, (size_t)n + 16);
    for (auto& c : build->cols) {
      BufPtr vb, bb;
      if (c.validity && n) { vb = dev_alloc(ctx, (size_t)n); SG_CUDA(launch_unpack_bits(static_cast<const uint8_t*>(c.validity->ptr), static_cast<uint8_t*>(vb->ptr), n, 0, ctx->stream)); }
      if (c.type.id == TypeId::Bool && n) { bb = dev_alloc(ctx, (size_t)n); SG_CUDA(launch_unpack_bits(static_cast<const uint8_t*>(c.data->ptr), static_cast<uint8_t*>(bb->ptr), n, 0, ctx->stream)); }
      build_valid_bytes.push_back(vb); build_bool_bytes.push_back(bb);
      if (c.type.is_string()) for (auto& h : c.heaps) build_heaps.push_back(h);
    }
    if (n == 0) return;
    brun.init(ctx, bs);
    brun.custom_sink = [this](PipelineCompiler& pc, CompiledPipeline& cp) { pc.finish_build(cp, lkeys); cp.extra_scratch = CHAIN_CACHE_BYTES; };
    auto cp = brun.compiled_for(*build);
    PipelineParams P;
    brun.prepare(P, *cp, *build, 0, n);
    PipelineAux aux; memset(&aux, 0, sizeof(aux));
    aux.build.table = static_cast<uint8_t*>(table->ptr);
    aux.build.capacity_mask = capacity - 1;
    aux.build.n_keys = (int)cp->keys.size();
    for (size_t i = 0; i < cp->keys.size(); ++i) aux.build.keys[i] = cp->keys[i];
    aux.build.row_base = 0;
    aux.build.dup_flag = static_cast<uint32_t*>(dupflag->ptr);
    aux.build.next = static_cast<int64_t*>(next->ptr);
    aux.build.smem_off = cp->scratch_off;
    for (size_t i = 0; i < lkeys.size(); ++i) {
      const DataType& kt = bs[(size_t)lkeys[i]].type;
      aux.build.key_cols[i] = static_cast<const uint8_t*>(build->cols[(size_t)lkeys[i]].data->ptr);
      aux.build.key_stride[i] = (uint8_t)(kt.is_string() ? 16 : kt.arrow_width());
    }
    brun.launch(P, cp, &aux, m);
    uint32_t d = 0;
    SG_CUDA(cudaMemcpyAsync(&d, dupflag->ptr, 4, cudaMemcpyDeviceToHost, ctx->stream));
    check_device_error(ctx, brun.scal.error());
    dup = d != 0;
  }

  // gathered build column `b` as a VM value (validity: gathered bytes AND `outer_valid` when given)
  Val gather_col(PipelineCompiler& pc, const Val& row, int b, const Val* outer_valid) {
    const DevColumn& c = build->cols[(size_t)b];
    const DataType t = bs[(size_t)b].type.storage();
    int idx = -1;
    Val v;
    auto set_ptr = [&](const void* p) { pc.prog()[(size_t)idx].imm1 = reinterpret_cast<uint64_t>(p); };
    switch (t.id) {
      case TypeId::Bool: v = pc.add_gather(row, K_B, 1, &idx); set_ptr(build_bool_bytes[(size_t)b]->ptr); break;
      case TypeId::Int32: case TypeId::Date32: v = pc.add_gather(row, K_I32, 4, &idx); set_ptr(c.data->ptr); break;
      case TypeId::Int64: case TypeId::UInt64: v = pc.add_gather(row, K_I64, 8, &idx); set_ptr(c.data->ptr); break;
      case TypeId::Float64: v = pc.add_gather(row, K_F64, 8, &idx); set_ptr(c.data->ptr); break;
      case TypeId::Decimal128:
        v = pc.add_gather(row, K_I128, 16, &idx); set_ptr(c.data->ptr);
        if (t.precision <= 18) { v.kind = K_I64; v.stride = 16; }
        break;
      case TypeId::Utf8: case TypeId::Utf8View: v = pc.add_gather(row, K_V16, 16, &idx); set_ptr(c.data->ptr); break;
      default: fail(SAILGPU_ERR_UNSUPPORTED, "join payload column of type " + t.str() + " is not supported yet");
    }
    Val valid; bool have = false;
    if (build_valid_bytes[(size_t)b]) {
      int vi = -1;
      valid = pc.add_gather(row, K_B, 1, &vi);
      pc.prog()[(size_t)vi].imm1 = reinterpret_cast<uint64_t>(build_valid_bytes[(size_t)b]->ptr);
      have = true;
    }
    if (outer_valid) { valid = have ? pc.and_val(valid, *outer_valid) : *outer_valid; have = true; }
    if (have) v.vslot = pc.materialize(valid).slot;
    return v;
  }

  void setup_probe_runner() {
    prun.init(ctx, ps);
    frun.init(ctx, joined);
    if (has_filter) {
      SG_CHECK(jt == "inner" || jt == "right_semi", SAILGPU_ERR_UNSUPPORTED, "residual join filter with join_type '" + jt + "' is not supported yet");
    }
    // which build columns does the output (projection / residual filter) touch?
    prun.pre_stages = [this](PipelineCompiler& pc, CompiledPipeline& cp) {
      pc.probe_params.push_back(&pp);
      auto mr = pc.add_probe(cp, rkeys, pp);
      const Val m_ = mr.first, row = mr.second;
      pp.table = static_cast<const uint8_t*>(table->ptr);
      pp.capacity_mask = capacity - 1;
      pp.visited = visited ? static_cast<uint8_t*>(visited->ptr) : nullptr;
      for (size_t i = 0; i < lkeys.size(); ++i) {
        pp.build_keys[i] = static_cast<const uint8_t*>(build->cols[(size_t)lkeys[i]].data->ptr);
        const DataType& kt = bs[(size_t)lkeys[i]].type;
        pp.build_stride[i] = (uint8_t)(kt.is_string() ? 16 : kt.arrow_width());
      }
      const int nb = (int)bs.size();
      if (jt == "inner" || jt == "right" || jt == "left") {
        std::vector<ExprPtr> nbind;
        for (int b = 0; b < nb; ++b) {
          ExprPtr ph = PipelineCompiler::placeholder(b, bs[(size_t)b].type, true);
          pc.bind_value(ph, gather_col(pc, row, b, jt == "right" ? &m_ : nullptr));
          nbind.push_back(ph);
        }
        for (auto& e : pc.bindings()) nbind.push_back(e);
        pc.bindings() = nbind;
        if (jt != "right") pc.and_mask(m_);
      } else if (jt == "right_semi") {
        if (has_filter) {
          std::vector<ExprPtr> probe_bind = pc.bindings(), nbind;
          for (int b = 0; b < nb; ++b) { ExprPtr ph = PipelineCompiler::placeholder(b, bs[(size_t)b].type, true); pc.bind_value(ph, gather_col(pc, row, b, nullptr)); nbind.push_back(ph); }
          for (auto& e : probe_bind) nbind.push_back(e);
          pc.bindings() = nbind;        // the filter stage sees build ++ probe; its projection maps back to probe columns
        }
        pc.and_mask(m_);
      } else if (jt == "right_anti") {
        pc.and_mask(pc.not_val(m_));
      } else {   // left_semi / left_anti: the probe only marks build rows; nothing is emitted here
        pc.and_mask(m_);
        pc.bindings().clear();
      }
    };
    // stages after the probe: residual filter and/or projection
    Schema cur = (jt == "right_semi" && has_filter) ? concat_schema() : joined;
    if (jt == "left_semi" || jt == "left_anti") return;
    if (has_filter) {
      StageSpec st; st.kind = StageSpec::Filter;
      st.predicate = parse_expr(filter_json, concat_schema());
      st.has_projection = true;
      if (jt == "right_semi") { for (size_t i = 0; i < ps.size(); ++i) if (!has_proj) st.projection.push_back((int)(bs.size() + i)); if (has_proj) for (int p : projection) st.projection.push_back((int)bs.size() + p); }
      else if (has_proj) st.projection = projection;
      else for (size_t i = 0; i < joined.size(); ++i) st.projection.push_back((int)i);
      prun.stages.push_back(st);
    } else if (has_proj) {
      StageSpec st; st.kind = StageSpec::Projection;
      for (int p : projection) { auto e = std::make_shared<Expr>(); e->kind = Expr::Col; e->col = p; e->type = joined[(size_t)p].type; e->nullable = true; st.exprs.push_back(e); st.names.push_back(joined[(size_t)p].name); }
      prun.stages.push_back(st);
    }
  }
  Schema concat_schema() const { Schema s = bs; for (auto& f : ps) s.push_back(f); return s; }

  bool runner_ready = false;

  void probe(const BatchPtr& b) {
    if (!runner_ready) { setup_probe_runner(); runner_ready = true; }
    if (build->rows == 0) {
      // empty build: inner/semi produce nothing; anti / right-outer pass every probe row
      if (jt == "right_anti") ready.push_back(project_plain(b, (int)0));
      else if (jt == "right") ready.push_back(right_outer_nulls(b));
      return;
    }
    if (b->rows == 0) return;
    if (swap_applies(*b)) { probe_swapped(b); return; }
    if (general_path()) { probe_general(b); return; }
    if (dup && (jt == "left_semi" || jt == "left_anti")) { mark_all_matches(b); return; }
    PipelineAux aux; memset(&aux, 0, sizeof(aux));
    // compile first (fills pp), then copy
    auto cpp = prun.compiled_for(*b);
    auto it = pps.find(cpp.get());
    if (it == pps.end()) it = pps.emplace(cpp.get(), pp).first;
    aux.probe[0] = it->second;
    BatchPtr out = run_streaming(prun, ctx, b, m, &aux, build_heaps);
    if (probe_streams_output() && out->rows > 0) ready.push_back(out);
  }

  // ---- duplicate-heavy build side met by a tiny probe batch: execute with the roles exchanged --------------------------
  // The duplicate path walks, for every probe row, the chain of build rows with its key -- one thread per probe row.  With
  // a handful of probe rows against millions of build rows (the plans put the growing intermediate on the build side:
  // TPC-H Q5 / Q7 join it with `nation`) that is a serial walk of ~10^6 dependent loads.  An inner join
  // is symmetric, so such a batch runs through a nested join that builds on the probe batch and streams the build side:
  // key pairs, residual filter and projection are re-indexed, the output schema is unchanged.  Output order follows the
  // streamed side (INTEGRATION.md: the join reports maintains_input_order = false).
  bool no_swap = false;
  bool swap_applies(const DevBatch& b) const {
    return !no_swap && dup && jt == "inner" && b.rows * 16 < build->rows;
  }
  static void remap_cols(Json& j, int nb, int np) {
    if (j.kind == Json::Obj) {
      for (auto& kv : j.o) {
        if (kv.first == "col" && kv.second.kind == Json::Num) {
          const int i = (int)kv.second.as_int();
          kv.second.s = std::to_string(i < nb ? i + np : i - nb);
        } else remap_cols(kv.second, nb, np);
      }
    } else if (j.kind == Json::Arr) {
      for (auto& x : j.a) remap_cols(x, nb, np);
    }
  }
  void probe_swapped(const BatchPtr& b) {
    const int nb = (int)bs.size(), np = (int)ps.size();
    auto sw = std::make_unique<JoinOp>();
    sw->ctx = ctx; sw->kind = "hash_join"; sw->in_schemas = {ps, bs};
    sw->bs = ps; sw->ps = bs; sw->jt = "inner"; sw->no_swap = true;
    sw->lkeys = rkeys; sw->rkeys = lkeys;
    sw->joined = ps;
    for (auto& f : bs) sw->joined.push_back(f);
    for (auto& f : sw->joined) f.nullable = true;
    if (has_filter) { sw->filter_json = filter_json; remap_cols(sw->filter_json, nb, np); sw->has_filter = true; }
    sw->has_proj = true;
    const int n_out = has_proj ? (int)projection.size() : nb + np;
    for (int k = 0; k < n_out; ++k) {
      const int j = has_proj ? projection[(size_t)k] : k;
      sw->projection.push_back(j < nb ? j + np : j - nb);
    }
    sw->out_schema = out_schema;
    sw->push(0, b);
    sw->finish(0);
    sw->push(1, build);
    sw->finish(1);
    for (;;) {
      BatchPtr o;
      const bool more = sw->pull(&o);
      if (o && o->rows > 0) ready.push_back(o);
      if (!more) break;
    }
    m.kernel_launches += sw->m.kernel_launches;
    m.pipeline_launches += sw->m.pipeline_launches;
    for (auto& pe : sw->m.pending) m.pending.push_back(pe);
    sw->m.pending.clear();
  }

  BatchPtr project_plain(const BatchPtr& b, int offset) {
    if (!has_proj) return b;
    auto out = std::make_shared<DevBatch>();
    out->rows = b->rows;
    for (int p : projection) out->cols.push_back(b->cols[(size_t)(p - offset)]);
    return out;
  }
  // right outer join against an empty build side: every probe row, build columns all NULL
  BatchPtr right_outer_nulls(const BatchPtr& b) {
    SG_CHECK(!has_filter, SAILGPU_ERR_UNSUPPORTED, "residual join filter with join_type 'right' is not supported yet");
    const int64_t n = b->rows;
    auto full = std::make_shared<DevBatch>();
    full->rows = n;
    for (auto& f : bs) {
      DevColumn c; c.type = f.type; c.length = n; c.arrow_is_utf8 = f.type.id == TypeId::Utf8;
      const size_t w = f.type.id == TypeId::Bool ? 0 : f.type.is_string() ? 16 : (size_t)f.type.arrow_width();
      c.data = dev_alloc_zero(ctx, w ? (size_t)n * w : (size_t)((n + 31) / 32 * 4));      // zero views = empty strings
      c.validity = dev_alloc_zero(ctx, (size_t)((n + 31) / 32 * 4));
      c.null_count = n;
      full->cols.push_back(c);
    }
    for (auto& c : b->cols) full->cols.push_back(c);
    if (!has_proj) return full;
    auto out = std::make_shared<DevBatch>();
    out->rows = n;
    for (int p : projection) out->cols.push_back(full->cols[(size_t)p]);
    return out;
  }

  // ---- duplicate build keys: count / scan / emit / gather ------------------------------------------
  void fill_raw(RawKeyCol* dst, const DevBatch& bt, const std::vector<int>& keys, const Schema& sch) {
    for (size_t i = 0; i < keys.size(); ++i) {
      const DevColumn& c = bt.cols[(size_t)keys[i]];
      const DataType& t = sch[(size_t)keys[i]].type;
      dst[i].data = static_cast<const uint8_t*>(c.data->ptr);
      dst[i].validity_bits = c.validity ? static_cast<const uint8_t*>(c.validity->ptr) : nullptr;
      dst[i].is_view = t.is_string() ? 1 : 0;
      const int w = t.is_string() ? 16 : t.arrow_width();
      SG_CHECK(w == 1 || w == 4 || w == 8 || w == 16, SAILGPU_ERR_UNSUPPORTED, "join key of type " + t.str() + " is not supported on the multi-match path");
      SG_CHECK(t.id != TypeId::Bool, SAILGPU_ERR_UNSUPPORTED, "boolean join keys are not supported");
      // the build sink packs <=18-digit decimals from their low 8 bytes; mirror that here
      dst[i].width = (t.is_decimal() && t.precision <= 18) ? 8 : w;
      dst[i].stride = w;
    }
  }

  DevColumn gather_column(const DevColumn& src, const Field& f, const int64_t* idx, int64_t n, bool idx_may_be_negative) {
    DevColumn c; c.type = f.type; c.length = n; c.arrow_is_utf8 = f.type.id == TypeId::Utf8; c.heaps = src.heaps;
    const bool bits = f.type.id == TypeId::Bool;
    if (bits) {
      BufPtr bytes = dev_alloc(ctx, (size_t)n + 4);
      SG_CUDA(launch_gather_bits(static_cast<const uint8_t*>(src.data->ptr), static_cast<uint8_t*>(bytes->ptr), idx, n, 0, ctx->stream));
      c.data = dev_alloc_zero(ctx, (size_t)((n + 31) / 32 * 4));
      SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(bytes->ptr), static_cast<uint32_t*>(c.data->ptr), n, nullptr, ctx->stream));
    } else {
      const int w = f.type.is_string() ? 16 : f.type.arrow_width();
      c.data = dev_alloc(ctx, (size_t)n * w);
      SG_CUDA(launch_gather_rows(static_cast<const uint8_t*>(src.data->ptr), static_cast<uint8_t*>(c.data->ptr), idx, n, w, ctx->stream));
    }
    if (src.validity || idx_may_be_negative) {
      BufPtr bytes = dev_alloc(ctx, (size_t)n + 4);
      SG_CUDA(launch_gather_bits(src.validity ? static_cast<const uint8_t*>(src.validity->ptr) : nullptr, static_cast<uint8_t*>(bytes->ptr), idx, n, 1, ctx->stream));
      c.validity = dev_alloc_zero(ctx, (size_t)((n + 31) / 32 * 4));
      SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(bytes->ptr), static_cast<uint32_t*>(c.validity->ptr), n, nullptr, ctx->stream));
      c.null_count = -1;
    }
    return c;
  }

  // duplicate build keys + a join that emits build rows: every matching build row must be marked
  void mark_all_matches(const BatchPtr& b) {
    JoinMultiParams J; memset(&J, 0, sizeof(J));
    J.n_probe = b->rows; J.n_keys = (int)lkeys.size();
    fill_raw(J.build_keys, *build, lkeys, bs);
    fill_raw(J.probe_keys, *b, rkeys, ps);
    J.table = static_cast<const uint8_t*>(table->ptr); J.capacity_mask = capacity - 1;
    J.visited = static_cast<uint8_t*>(visited->ptr);
    J.next = static_cast<const int64_t*>(next->ptr);
    J.pass = 2;
    SG_CUDA(launch_join_multi(J, ctx->stream));
    m.kernel_launches++;
  }

  void probe_general(const BatchPtr& b) {
    const int64_t n = b->rows;
    JoinMultiParams J; memset(&J, 0, sizeof(J));
    J.n_probe = n; J.n_keys = (int)lkeys.size();
    fill_raw(J.build_keys, *build, lkeys, bs);
    fill_raw(J.probe_keys, *b, rkeys, ps);
    J.table = static_cast<const uint8_t*>(table->ptr); J.capacity_mask = capacity - 1;
    J.emit_unmatched_probe = jt == "right" ? 1 : 0;
    J.next = static_cast<const int64_t*>(next->ptr);
    BufPtr counts = dev_alloc(ctx, (size_t)n * 4), offs = dev_alloc(ctx, (size_t)n * 8), scratch = dev_alloc(ctx, 1026 * 8);
    J.counts = static_cast<uint32_t*>(counts->ptr); J.pass = 0;
    SG_CUDA(launch_join_multi(J, ctx->stream));
    SG_CUDA(launch_exclusive_scan_u32(J.counts, n, static_cast<uint64_t*>(offs->ptr), static_cast<uint64_t*>(scratch->ptr), ctx->stream));
    const int64_t nblocks = std::min<int64_t>(1024, (n + 4095) / 4096);
    uint64_t total = 0;
    SG_CUDA(cudaMemcpyAsync(&total, static_cast<uint64_t*>(scratch->ptr) + nblocks, 8, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    if (total == 0) return;
    BufPtr ob = dev_alloc(ctx, (size_t)total * 8), op = dev_alloc(ctx, (size_t)total * 8);
    J.offsets = static_cast<const uint64_t*>(offs->ptr); J.out_build = static_cast<int64_t*>(ob->ptr); J.out_probe = static_cast<int64_t*>(op->ptr);
    J.visited = visited ? static_cast<uint8_t*>(visited->ptr) : nullptr;
    J.pass = 1;
    SG_CUDA(launch_join_multi(J, ctx->stream));
    m.kernel_launches += 2;
    auto out = std::make_shared<DevBatch>();
    out->rows = (int64_t)total;
    for (size_t i = 0; i < bs.size(); ++i) out->cols.push_back(gather_column(build->cols[i], bs[i], J.out_build, (int64_t)total, jt == "right"));
    for (size_t i = 0; i < ps.size(); ++i) out->cols.push_back(gather_column(b->cols[i], ps[i], J.out_probe, (int64_t)total, false));
    stream_sync(ctx);
    ready.push_back(post_filter(out));
  }

  // residual filter / projection over a materialised joined batch
  BatchPtr post_filter(const BatchPtr& joined_batch) {
    if (!has_filter && !has_proj) return joined_batch;
    if (frun.stages.empty()) {
      if (has_filter) {
        StageSpec st; st.kind = StageSpec::Filter; st.predicate = parse_expr(filter_json, joined); st.has_projection = has_proj; st.projection = projection;
        frun.stages.push_back(st);
      } else {
        return project_plain(joined_batch, 0);
      }
    }
    return run_streaming(frun, ctx, joined_batch, m, nullptr, {});
  }

  // ---- end of probe: rows that come from the build side -------------------------------------------
  void emit_tail() {
    if (tail_done) return;
    tail_done = true;
    if (!needs_visited() || build->rows == 0) return;
    const int64_t n = build->rows;
    auto ext = std::make_shared<DevBatch>(*build);
    DevColumn vis; vis.type = T(TypeId::Bool); vis.length = n;
    vis.data = dev_alloc_zero(ctx, (size_t)((n + 31) / 32 * 4));
    SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(visited->ptr), static_cast<uint32_t*>(vis.data->ptr), n, nullptr, ctx->stream));
    ext->cols.push_back(vis);
    Schema es = bs; es.push_back({"__visited", T(TypeId::Bool), false});
    trun.init(ctx, es);
    auto vcol = std::make_shared<Expr>(); vcol->kind = Expr::Col; vcol->col = (int)bs.size(); vcol->type = T(TypeId::Bool);
    ExprPtr pred = vcol;
    if (jt != "left_semi") { auto nt = std::make_shared<Expr>(); nt->kind = Expr::Not; nt->args = {vcol}; nt->type = T(TypeId::Bool); pred = nt; }
    StageSpec f; f.kind = StageSpec::Filter; f.predicate = pred; f.has_projection = true;
    for (size_t i = 0; i < bs.size(); ++i) f.projection.push_back((int)i);
    trun.stages.push_back(f);
    if (jt == "left") {           // unmatched build rows ++ NULL probe columns
      StageSpec p; p.kind = StageSpec::Projection;
      for (size_t i = 0; i < bs.size(); ++i) { auto e = std::make_shared<Expr>(); e->kind = Expr::Col; e->col = (int)i; e->type = bs[i].type; e->nullable = true; p.exprs.push_back(e); p.names.push_back(bs[i].name); }
      for (auto& fld : ps) { auto e = std::make_shared<Expr>(); e->kind = Expr::Lit; e->type = fld.type; e->lit_null = true; e->nullable = true; p.exprs.push_back(e); p.names.push_back(fld.name); }
      trun.stages.push_back(p);
    }
    if (has_proj) {
      StageSpec p; p.kind = StageSpec::Projection;
      for (int q : projection) { auto e = std::make_shared<Expr>(); e->kind = Expr::Col; e->col = q; e->type = joined[(size_t)q].type; e->nullable = true; p.exprs.push_back(e); p.names.push_back(joined[(size_t)q].name); }
      trun.stages.push_back(p);
    }
    BatchPtr out = run_streaming(trun, ctx, ext, m, nullptr, {});
    if (out->rows > 0) ready.push_back(out);
  }
};

static std::unique_ptr<Op> make_plain_join_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs) {
  SG_CHECK(inputs.size() == 2, SAILGPU_ERR_INVALID, "hash_join takes two inputs (build = left, probe = right)");
  auto op = std::make_unique<JoinOp>();
  op->ctx = ctx; op->kind = "hash_join"; op->in_schemas = inputs;
  op->bs = inputs[0]; op->ps = inputs[1];
  const Json* jtj = spec.find("join_type");
  op->jt = jtj ? jtj->as_str() : "inner";
  static const char* known[] = {"inner", "left", "right", "left_semi", "left_anti", "right_semi", "right_anti"};
  bool ok = false; for (auto k : known) ok |= op->jt == k;
  SG_CHECK(ok, SAILGPU_ERR_UNSUPPORTED, "join_type '" + op->jt + "' is not supported on the GPU path yet");
  for (auto& pr : spec.at("on").a) {
    SG_CHECK(pr.kind == Json::Arr && pr.a.size() == 2, SAILGPU_ERR_INVALID, "hash_join 'on' entries must be [left_col, right_col]");
    const int l = (int)pr.a[0].as_int(), r = (int)pr.a[1].as_int();
    SG_CHECK(l >= 0 && l < (int)op->bs.size() && r >= 0 && r < (int)op->ps.size(), SAILGPU_ERR_INVALID, "join key index out of range");
    DataType lt = op->bs[(size_t)l].type, rt = op->ps[(size_t)r].type;
    SG_CHECK(lt == rt || (lt.is_string() && rt.is_string()), SAILGPU_ERR_UNSUPPORTED, "join keys " + lt.str() + " / " + rt.str() + " differ in type");
    op->lkeys.push_back(l); op->rkeys.push_back(r);
  }
  SG_CHECK(!op->lkeys.empty() && (int)op->lkeys.size() <= MAX_KEYS, SAILGPU_ERR_INVALID, "hash_join needs 1.." + std::to_string(MAX_KEYS) + " key pairs");
  const Json* nen = spec.find("null_equals_null");
  SG_CHECK(!(nen && nen->kind == Json::Bool && nen->b), SAILGPU_ERR_UNSUPPORTED, "null_equals_null joins are not supported yet");
  if (op->jt == "left_semi" || op->jt == "left_anti") op->joined = op->bs;
  else if (op->jt == "right_semi" || op->jt == "right_anti") op->joined = op->ps;
  else {
    op->joined = op->bs;
    for (auto& f : op->ps) op->joined.push_back(f);
    for (auto& f : op->joined) f.nullable = true;
  }
  const Json* fj = spec.find("filter");
  if (fj && !fj->is_null()) { op->filter_json = *fj; op->has_filter = true; }
  // data-independent limits are reported here, at plan time (sailgpu_spec_validate), never after the build side was consumed
  SG_CHECK(!op->has_filter || op->jt == "inner" || op->jt == "right_semi" || op->jt == "left_semi" || op->jt == "left_anti", SAILGPU_ERR_UNSUPPORTED,
           "residual join filter with join_type '" + op->jt + "' is not supported yet");
  for (size_t i = 0; i < op->lkeys.size(); ++i) {
    const DataType& t = op->bs[(size_t)op->lkeys[i]].type;
    SG_CHECK(t.id != TypeId::Bool, SAILGPU_ERR_UNSUPPORTED, "boolean join keys are not supported");
    const int w = t.is_string() ? 16 : t.arrow_width();
    SG_CHECK(w == 1 || w == 4 || w == 8 || w == 16, SAILGPU_ERR_UNSUPPORTED, "join key of type " + t.str() + " is not supported");
  }
  const Json* pj = spec.find("projection");
  if (pj && !pj->is_null()) {
    op->has_proj = true;
    for (auto& x : pj->a) { const int i = (int)x.as_int(); SG_CHECK(i >= 0 && i < (int)op->joined.size(), SAILGPU_ERR_INVALID, "join projection index out of range"); op->projection.push_back(i); }
  }
  if (op->has_proj) for (int i : op->projection) op->out_schema.push_back(op->joined[(size_t)i]);
  else op->out_schema = op->joined;
  return op;
}

// ================================================================================================
// LeftSemi / LeftAnti joins WITH a residual filter (TPC-H Q21: `exists (.. l2.l_suppkey <> l1.l_suppkey)`,
// test_tpch.plan.yaml:621-622).  A build row qualifies when SOME key-matching probe row passes the filter, so matches have
// to be enumerated as pairs.  Composed from the two joins the library already has: the build side gets a row-number column;
// an inner join with the filter yields the row numbers of the build rows that found a partner; a filter-less semi / anti
// join of the build side against those numbers emits the result.
// ================================================================================================
struct FilteredSemiJoinOp : Op {
  std::unique_ptr<Op> pairs, pick;
  std::vector<BatchPtr> bparts;
  std::deque<BatchPtr> ready;
  bool build_done = false, probe_done = false, finished = false;

  static Json jnum(int64_t v) { Json j; j.kind = Json::Num; j.s = std::to_string(v); return j; }
  static Json jstr(const std::string& v) { Json j; j.kind = Json::Str; j.s = v; return j; }
  static Json jarr(std::vector<Json> v) { Json j; j.kind = Json::Arr; j.a = std::move(v); return j; }

  void drain(Op& from, Op* to) {
    for (;;) {
      BatchPtr b;
      const bool more = from.pull(&b);
      if (b && b->rows > 0) { if (to) to->push(1, b); else ready.push_back(b); }
      if (!b || !more) break;
    }
  }
  void push(int input, const BatchPtr& b) override {
    if (input == 0) { SG_CHECK(!build_done, SAILGPU_ERR_STATE, "build input already finished"); bparts.push_back(b); m.build_input_rows += (uint64_t)b->rows; m.build_input_batches++; return; }
    SG_CHECK(input == 1 && build_done, input == 1 ? SAILGPU_ERR_STATE : SAILGPU_ERR_INVALID, "hash_join: the build input must be finished before the probe input is pushed");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    pairs->push(1, b);
    drain(*pairs, pick.get());
  }
  void finish(int input) override {
    if (input == 0) {
      const Schema& bs = in_schemas[0];
      BatchPtr build = bparts.empty() ? empty_batch(ctx, bs) : concat_batches(ctx, bs, bparts);
      bparts.clear();
      auto with_id = std::make_shared<DevBatch>(*build);
      DevColumn id; id.type = T(TypeId::Int64); id.length = build->rows;
      id.data = dev_alloc(ctx, (size_t)build->rows * 8);
      SG_CUDA(launch_iota(static_cast<int64_t*>(id.data->ptr), build->rows, ctx->stream));
      with_id->cols.push_back(id);
      pairs->push(0, with_id); pairs->finish(0);
      pick->push(0, with_id); pick->finish(0);
      build_done = true;
      return;
    }
    probe_done = true;
    pairs->finish(1);
    drain(*pairs, pick.get());
    pick->finish(1);
    drain(*pick, nullptr);
    finished = true;
    m.kernel_launches += pairs->m.kernel_launches + pick->m.kernel_launches;
  }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (!ready.empty()) { *out = ready.front(); ready.pop_front(); m.output_rows += (uint64_t)(*out)->rows; m.output_batches++; }
    return !ready.empty() || !finished;
  }
};

// ================================================================================================
// LeftSemi / LeftAnti without a residual filter: DataFusion builds on the LEFT input whatever its size (CollectLeft), and TPC-H
// Q18 / Q20 put a 60 M-row join result there against a probe side of a few dozen keys -- 6.4 ms of hash-table build at SF10 for a
// 99-row probe.  Both inputs of these join types are complete before a single row can be emitted (the build rows come out after
// the last probe batch), so the operator waits: probe batches are held while they stay below 1/8 of the build side, and if the
// probe input ends that small the ROLES ARE EXCHANGED -- hash table on the probe keys, the big side streamed through a
// RightSemi / RightAnti probe (same rows: a row of the left input qualifies iff its key has / has no partner on the right).
// Otherwise the plain operator runs exactly as before.
// ================================================================================================
struct LazySemiJoinOp : Op {
  Json spec;
  std::unique_ptr<Op> inner;          // set once the decision is taken
  std::vector<BatchPtr> bparts, pparts;
  int64_t build_rows = 0, probe_rows = 0;
  bool build_done = false, finished = false;
  std::deque<BatchPtr> ready;

  void drain() {
    for (;;) {
      BatchPtr b;
      const bool more = inner->pull(&b);
      if (b && b->rows > 0) ready.push_back(b);
      if (!b || !more) break;
    }
  }
  void commit_plain() {
    inner = make_plain_join_op(ctx, spec, in_schemas);
    for (auto& b : bparts) inner->push(0, b);
    inner->finish(0);
    bparts.clear();
    for (auto& b : pparts) inner->push(1, b);
    pparts.clear();
  }
  void push(int input, const BatchPtr& b) override {
    if (input == 0) {
      SG_CHECK(!build_done, SAILGPU_ERR_STATE, "build input already finished");
      m.build_input_rows += (uint64_t)b->rows; m.build_input_batches++;
      bparts.push_back(b); build_rows += b->rows;
      return;
    }
    SG_CHECK(input == 1 && build_done, input == 1 ? SAILGPU_ERR_STATE : SAILGPU_ERR_INVALID, "hash_join: the build input must be finished before the probe input is pushed");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    if (inner) { inner->push(1, b); return; }
    pparts.push_back(b); probe_rows += b->rows;
    if (probe_rows * 8 >= build_rows) commit_plain();          // not a small probe side: the plain operator takes over
  }
  void finish(int input) override {
    if (input == 0) { build_done = true; return; }
    if (!inner) {
      // roles exchanged: {on: [[probe key, build key]], RightSemi/RightAnti}; the projection indexes the left input's columns in both forms
      const std::string jt = spec.at("join_type").as_str();
      std::vector<std::pair<std::string, Json>> o;
      for (auto& kv : spec.o) {
        if (kv.first == "join_type") { Json j; j.kind = Json::Str; j.s = jt == "left_semi" ? "right_semi" : "right_anti"; o.push_back({"join_type", j}); }
        else if (kv.first == "on") {
          Json on; on.kind = Json::Arr;
          for (auto& pr : kv.second.a) { Json x; x.kind = Json::Arr; x.a = {pr.a[1], pr.a[0]}; on.a.push_back(x); }
          o.push_back({"on", on});
        } else o.push_back(kv);
      }
      Json sw; sw.kind = Json::Obj; sw.o = o;
      inner = make_plain_join_op(ctx, sw, {in_schemas[1], in_schemas[0]});
      for (auto& b : pparts) inner->push(0, b);
      inner->finish(0);
      pparts.clear();
      for (auto& b : bparts) { inner->push(1, b); drain(); }
      bparts.clear();
      inner->finish(1);
    } else inner->finish(1);
    drain();
    finished = true;
    m.kernel_launches += inner->m.kernel_launches;
  }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (!ready.empty()) { *out = ready.front(); ready.pop_front(); m.output_rows += (uint64_t)(*out)->rows; m.output_batches++; }
    return !ready.empty() || !finished;
  }
};

std::unique_ptr<Op> make_join_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs) {
  SG_CHECK(inputs.size() == 2, SAILGPU_ERR_INVALID, "hash_join takes two inputs (build = left, probe = right)");
  const Json* jtj = spec.find("join_type");
  const std::string jt = jtj ? jtj->as_str() : "inner";
  const Json* fj = spec.find("filter");
  if ((jt == "left_semi" || jt == "left_anti") && !(fj && !fj->is_null())) {
    auto plain = make_plain_join_op(ctx, spec, inputs);     // plan-time validation + output schema
    auto op = std::make_unique<LazySemiJoinOp>();
    op->ctx = ctx; op->kind = "hash_join"; op->in_schemas = inputs; op->out_schema = plain->out_schema; op->spec = spec;
    return op;
  }
  if (!((jt == "left_semi" || jt == "left_anti") && fj && !fj->is_null())) return make_plain_join_op(ctx, spec, inputs);
  // validates keys / projection / filter types exactly as the plain operator would (its output schema is ours)
  auto plain = make_plain_join_op(ctx, spec, inputs);
  auto op = std::make_unique<FilteredSemiJoinOp>();
  op->ctx = ctx; op->kind = "hash_join"; op->in_schemas = inputs; op->out_schema = plain->out_schema;
  (void)parse_expr(*fj, [&] { Schema s = inputs[0]; for (auto& f : inputs[1]) s.push_back(f); return s; }());
  const int nb = (int)inputs[0].size();
  Schema bs_id = inputs[0];
  bs_id.push_back({"__row", T(TypeId::Int64), false});
  // (a) inner join with the filter; columns of (build ++ __row ++ probe): probe column j sits at nb + 1 + j
  Json fmap = *fj;
  std::function<void(Json&)> shift = [&](Json& j) {
    if (j.kind == Json::Obj) {
      for (auto& kv : j.o) {
        if (kv.first == "col" && kv.second.kind == Json::Num) { const int i = (int)kv.second.as_int(); if (i >= nb) kv.second.s = std::to_string(i + 1); }
        else shift(kv.second);
      }
    } else if (j.kind == Json::Arr) for (auto& x : j.a) shift(x);
  };
  shift(fmap);
  Json a; a.kind = Json::Obj;
  a.o = {{"op", FilteredSemiJoinOp::jstr("hash_join")}, {"join_type", FilteredSemiJoinOp::jstr("inner")}, {"on", spec.at("on")}, {"filter", fmap},
         {"projection", FilteredSemiJoinOp::jarr({FilteredSemiJoinOp::jnum(nb)})}};
  op->pairs = make_plain_join_op(ctx, a, {bs_id, inputs[1]});
  // (b) semi / anti join of the build side against the row numbers that found a partner
  std::vector<Json> proj;
  const Json* pj = spec.find("projection");
  if (pj && !pj->is_null()) for (auto& x : pj->a) proj.push_back(x);
  else for (int i = 0; i < nb; ++i) proj.push_back(FilteredSemiJoinOp::jnum(i));
  Json b; b.kind = Json::Obj;
  b.o = {{"op", FilteredSemiJoinOp::jstr("hash_join")}, {"join_type", FilteredSemiJoinOp::jstr(jt)},
         {"on", FilteredSemiJoinOp::jarr({FilteredSemiJoinOp::jarr({FilteredSemiJoinOp::jnum(nb), FilteredSemiJoinOp::jnum(0)})})},
         {"projection", FilteredSemiJoinOp::jarr(proj)}};
  Schema ids = {{"__row", T(TypeId::Int64), true}};
  op->pick = make_plain_join_op(ctx, b, {bs_id, ids});
  return op;
}

// ================================================================================================
// NestedLoopJoinExec (inner) with a small build side: what DataFusion plans for the scalar-subquery shapes of TPC-H Q11 /
// Q22 (test_tpch.plan.yaml:333,661 -- the left child is a one-row aggregate).  Every build row turns into literals of a
// Filter -> Projection pipeline over the probe batches, so the join is one pass of the tile pipeline per build row and
// inherits its expression support (and its specialised kernels).  Build sides beyond a few dozen rows are refused.
// ================================================================================================
struct NestedLoopJoinOp : Op {
  static constexpr int64_t MAX_BUILD_ROWS = 64;
  Schema ls, rs, joined;
  ExprPtr filter;                     // over `joined` (left ++ right); null: cross join
  std::vector<int> projection;        // into `joined`
  std::vector<BatchPtr> lparts;
  std::vector<std::unique_ptr<PipelineRunner>> runs;   // one per build row
  std::deque<BatchPtr> pending, ready;
  bool left_done = false, right_done = false;

  static ExprPtr literal_of(Ctx* ctx, const DevColumn& c, const DataType& t, int64_t row) {
    auto e = std::make_shared<Expr>();
    e->kind = Expr::Lit; e->type = t;
    if (c.validity) {
      uint8_t byte = 0;
      SG_CUDA(cudaMemcpyAsync(&byte, static_cast<const uint8_t*>(c.validity->ptr) + (row >> 3), 1, cudaMemcpyDeviceToHost, ctx->stream));
      stream_sync(ctx);
      if (!((byte >> (row & 7)) & 1)) { e->lit_null = true; e->nullable = true; return e; }
    }
    if (t.id == TypeId::Bool) {
      uint8_t byte = 0;
      SG_CUDA(cudaMemcpyAsync(&byte, static_cast<const uint8_t*>(c.data->ptr) + (row >> 3), 1, cudaMemcpyDeviceToHost, ctx->stream));
      stream_sync(ctx);
      e->lit_i = (byte >> (row & 7)) & 1;
      return e;
    }
    const int w = t.is_string() ? 16 : t.arrow_width();
    uint8_t raw[16] = {0};
    SG_CUDA(cudaMemcpyAsync(raw, static_cast<const uint8_t*>(c.data->ptr) + row * w, (size_t)w, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    if (t.is_string()) {
      uint32_t len; memcpy(&len, raw, 4);
      e->lit_s.resize(len);
      if (len <= 12) memcpy(&e->lit_s[0], raw + 4, len);
      else {
        uint64_t ptr; memcpy(&ptr, raw + 8, 8);       // resolved view: absolute device pointer
        SG_CUDA(cudaMemcpyAsync(&e->lit_s[0], reinterpret_cast<const void*>(ptr), len, cudaMemcpyDeviceToHost, ctx->stream));
        stream_sync(ctx);
      }
    } else if (t.id == TypeId::Float64) { memcpy(&e->lit_f, raw, 8); }
    else if (t.id == TypeId::Float32) { float f; memcpy(&f, raw, 4); e->lit_f = f; }
    else if (w == 16) { u128 v; memcpy(&v, raw, 16); e->lit_i = (i128)v; }
    else if (w == 8) { int64_t v; memcpy(&v, raw, 8); e->lit_i = t.is_unsigned_int() ? (i128)(uint64_t)v : (i128)v; }
    else if (w == 4) { int32_t v; memcpy(&v, raw, 4); e->lit_i = t.is_unsigned_int() ? (i128)(uint32_t)v : (i128)v; }
    else if (w == 2) { int16_t v; memcpy(&v, raw, 2); e->lit_i = t.is_unsigned_int() ? (i128)(uint16_t)v : (i128)v; }
    else { int8_t v; memcpy(&v, raw, 1); e->lit_i = t.is_unsigned_int() ? (i128)(uint8_t)v : (i128)v; }
    return e;
  }
  // expression over (left ++ right) -> expression over right with the build row's values as literals
  ExprPtr bind_row(const ExprPtr& e, const std::vector<ExprPtr>& lits) const {
    if (e->kind == Expr::Col) {
      if (e->col < (int)ls.size()) return lits[(size_t)e->col];
      auto c = std::make_shared<Expr>(*e);
      c->col = e->col - (int)ls.size();
      return c;
    }
    if (e->kind == Expr::Lit) return e;
    auto c = std::make_shared<Expr>(*e);
    for (auto& a : c->args) a = bind_row(a, lits);
    return c;
  }

  void build_runners() {
    BatchPtr left = lparts.empty() ? empty_batch(ctx, ls) : concat_batches(ctx, ls, lparts);
    lparts.clear();
    SG_CHECK(left->rows <= MAX_BUILD_ROWS, SAILGPU_ERR_UNSUPPORTED,
             "nested loop join with " + std::to_string(left->rows) + " build rows (the GPU path covers the scalar-subquery shapes: at most " + std::to_string(MAX_BUILD_ROWS) + ")");
    for (int64_t r = 0; r < left->rows; ++r) {
      std::vector<ExprPtr> lits;
      for (size_t c = 0; c < ls.size(); ++c) lits.push_back(literal_of(ctx, left->cols[c], ls[c].type, r));
      auto run = std::make_unique<PipelineRunner>();
      run->init(ctx, rs);
      if (filter) { StageSpec f; f.kind = StageSpec::Filter; f.predicate = bind_row(filter, lits); run->stages.push_back(f); }
      StageSpec p; p.kind = StageSpec::Projection;
      for (size_t k = 0; k < projection.size(); ++k) {
        const int j = projection[k];
        ExprPtr e;
        if (j < (int)ls.size()) e = lits[(size_t)j];
        else { e = std::make_shared<Expr>(); e->kind = Expr::Col; e->col = j - (int)ls.size(); e->type = rs[(size_t)e->col].type; e->nullable = rs[(size_t)e->col].nullable; }
        p.exprs.push_back(e); p.names.push_back(out_schema[k].name);
      }
      run->stages.push_back(p);
      runs.push_back(std::move(run));
    }
  }
  void probe(const BatchPtr& b) {
    if (b->rows == 0) return;
    for (auto& run : runs) {
      BatchPtr out = run_streaming(*run, ctx, b, m, nullptr, {});
      if (out->rows > 0) ready.push_back(out);
    }
  }
  void push(int input, const BatchPtr& b) override {
    const uint64_t t0 = now_ns();
    if (input == 0) { SG_CHECK(!left_done, SAILGPU_ERR_STATE, "build input already finished"); lparts.push_back(b); m.build_input_rows += (uint64_t)b->rows; m.build_input_batches++; return; }
    SG_CHECK(input == 1, SAILGPU_ERR_INVALID, "nested_loop_join has two inputs");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    if (!left_done) { pending.push_back(b); return; }
    probe(b);
    m.elapsed_compute_ns += now_ns() - t0;
  }
  void finish(int input) override {
    if (input == 0) {
      left_done = true;
      build_runners();
      while (!pending.empty()) { probe(pending.front()); pending.pop_front(); }
    } else right_done = true;
  }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (!ready.empty()) { *out = ready.front(); ready.pop_front(); m.output_rows += (uint64_t)(*out)->rows; m.output_batches++; }
    return !ready.empty() || !(left_done && right_done);
  }
};

std::unique_ptr<Op> make_nlj_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs) {
  SG_CHECK(inputs.size() == 2, SAILGPU_ERR_INVALID, "nested_loop_join takes two inputs (build = left, probe = right)");
  auto op = std::make_unique<NestedLoopJoinOp>();
  op->ctx = ctx; op->kind = "nested_loop_join"; op->in_schemas = inputs;
  op->ls = inputs[0]; op->rs = inputs[1];
  const Json* jt = spec.find("join_type");
  SG_CHECK(!jt || jt->as_str() == "inner", SAILGPU_ERR_UNSUPPORTED, "nested_loop_join: only join_type 'inner' runs on the GPU path");
  op->joined = op->ls;
  for (auto& f : op->rs) op->joined.push_back(f);
  const Json* fj = spec.find("filter");
  if (fj && !fj->is_null()) {
    op->filter = parse_expr(*fj, op->joined);
    SG_CHECK(op->filter->type.id == TypeId::Bool, SAILGPU_ERR_INVALID, "join filter must be boolean");
  }
  const Json* pj = spec.find("projection");
  if (pj && !pj->is_null()) {
    for (auto& x : pj->a) { const int i = (int)x.as_int(); SG_CHECK(i >= 0 && i < (int)op->joined.size(), SAILGPU_ERR_INVALID, "join projection index out of range"); op->projection.push_back(i); }
  } else for (size_t i = 0; i < op->joined.size(); ++i) op->projection.push_back((int)i);
  for (int i : op->projection) op->out_schema.push_back(op->joined[(size_t)i]);
  // the joined rows are written by a streaming pipeline: its limit, reported while planning
  SG_CHECK((int)op->out_schema.size() <= MAX_OUTPUTS, SAILGPU_ERR_UNSUPPORTED, "nested_loop_join: more than " + std::to_string(MAX_OUTPUTS) + " output columns");
  return op;
}

// ================================================================================================
// SortExec (+ TopK)
// ================================================================================================
// scratch of radix_sort_indices for n rows; `hold` keeps its buffers
static RadixScratch radix_scratch(Ctx* ctx, int64_t n, std::vector<BufPtr>& hold) {
  const int64_t n_chunks = (n + 2047) / 2048;
  auto buf = [&](size_t bytes) { hold.push_back(dev_alloc(ctx, bytes)); return hold.back()->ptr; };
  RadixScratch S;
  S.idx_a = static_cast<uint32_t*>(buf((size_t)n * 4)); S.idx_b = static_cast<uint32_t*>(buf((size_t)n * 4));
  S.kw_a = static_cast<uint64_t*>(buf((size_t)n * 8)); S.kw_b = static_cast<uint64_t*>(buf((size_t)n * 8));
  S.hist = static_cast<uint32_t*>(buf((size_t)n_chunks * 256 * 4)); S.offs = static_cast<uint64_t*>(buf((size_t)n_chunks * 256 * 8));
  S.scan_scratch = static_cast<uint64_t*>(buf(1026 * 8));
  return S;
}

struct SortOp : Op {
  struct Key { ExprPtr e; bool asc, nulls_first; };
  std::vector<Key> keys;
  int64_t fetch = -1;
  std::vector<BatchPtr> parts;
  bool input_done = false, emitted = false;
  PipelineRunner krun;       // evaluates non-column sort expressions

  void push(int input, const BatchPtr& b) override {
    SG_CHECK(input == 0, SAILGPU_ERR_INVALID, "sort has one input");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    parts.push_back(b);
  }
  void finish(int) override { input_done = true; }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (!input_done) return true;
    if (emitted) return false;
    const uint64_t t0 = now_ns();
    *out = run();
    emitted = true;
    m.elapsed_compute_ns += now_ns() - t0;
    m.output_rows += (uint64_t)(*out)->rows; m.output_batches++;
    return false;
  }

  struct Encoded { BufPtr keys, bits; int key_bytes = 0; std::vector<BufPtr> ranks; };

  // the key columns of every row as the encoder, the small sort and the TopK selection read them (string keys: no ranks yet)
  SortEncodeParams describe_keys(const BatchPtr& all, const Schema& sch, const std::vector<Key>& ks) {
    SortEncodeParams E; memset(&E, 0, sizeof(E));
    E.n = all->rows; E.n_keys = (int)ks.size();
    SG_CHECK(ks.size() <= sizeof(E.cols) / sizeof(E.cols[0]), SAILGPU_ERR_UNSUPPORTED, "more than 8 sort keys");
    for (size_t k = 0; k < ks.size(); ++k) {
      SG_CHECK(ks[k].e->kind == Expr::Col, SAILGPU_ERR_UNSUPPORTED, "sort keys must be column references");
      const DevColumn& c = all->cols[(size_t)ks[k].e->col];
      const DataType t = sch[(size_t)ks[k].e->col].type.storage();
      SortKeyCol& s = E.cols[k];
      s.data = static_cast<const uint8_t*>(c.data->ptr);
      s.validity_bits = c.validity ? static_cast<const uint8_t*>(c.validity->ptr) : nullptr;
      s.asc = ks[k].asc; s.nulls_first = ks[k].nulls_first;
      if (t.is_string()) { s.kind = SORT_VIEW; s.width = 16; s.enc_bytes = 4; }
      else if (t.id == TypeId::Bool) { s.kind = SORT_BOOL; s.width = 1; s.enc_bytes = 1; }
      else if (t.is_float()) { SG_CHECK(t.id == TypeId::Float64, SAILGPU_ERR_UNSUPPORTED, "Float32 sort keys"); s.kind = SORT_F64; s.width = 8; s.enc_bytes = 8; }
      else if (t.is_unsigned_int()) { s.kind = SORT_UINT; s.width = t.arrow_width(); s.enc_bytes = s.width; }
      else { s.kind = SORT_INT; s.width = t.arrow_width(); s.enc_bytes = s.width; }
    }
    return E;
  }

  // the dense rank of every row's string in a string key column (string_ranks, relational.cu)
  BufPtr string_ranks_of(const SortKeyCol& c, int64_t n) {
    std::vector<BufPtr> hold;
    auto buf = [&](size_t bytes) { hold.push_back(dev_alloc(ctx, bytes)); return hold.back()->ptr; };
    StringRankScratch S;
    S.radix = radix_scratch(ctx, n, hold);
    S.keys = static_cast<uint8_t*>(buf((size_t)n * 13));
    S.perm = static_cast<uint32_t*>(buf((size_t)n * 4)); S.head = static_cast<uint32_t*>(buf((size_t)n * 4)); S.rowof = static_cast<uint32_t*>(buf((size_t)n * 4));
    for (int i = 0; i < 2; ++i) { S.opos[i] = static_cast<uint32_t*>(buf((size_t)n * 4)); S.grp[i] = static_cast<uint32_t*>(buf((size_t)n * 4)); }
    S.flags = static_cast<uint64_t*>(buf((size_t)n * 8)); S.before = static_cast<uint64_t*>(buf((size_t)n * 8));
    S.scan_scratch = static_cast<uint64_t*>(buf(1026 * 8));
    S.ctrl = static_cast<uint32_t*>(buf(32 * 4));
    BufPtr rank = dev_alloc(ctx, (size_t)n * 4);
    int launches = 0, syncs = 0;
    SG_CUDA(string_ranks(c.data, c.validity_bits, n, static_cast<uint32_t*>(rank->ptr), S, ctx->stream, &launches, &syncs));
    m.kernel_launches += (uint64_t)launches;
    ctx->host_syncs += (uint64_t)syncs;
    return rank;
  }

  // order-preserving fixed-width encoding of the sort keys of every row (memcmp order == requested order).  A string key is its
  // null byte and its 4-byte dense rank among the rows, so the width does not depend on the strings' lengths.
  Encoded encode_keys(const BatchPtr& all, const Schema& sch, const std::vector<Key>& ks) {
    const int64_t n = all->rows;
    SortEncodeParams E = describe_keys(all, sch, ks);
    Encoded out;
    int off = 0;
    for (size_t k = 0; k < ks.size(); ++k) {
      if (E.cols[k].kind == SORT_VIEW) { out.ranks.push_back(string_ranks_of(E.cols[k], n)); E.cols[k].rank = static_cast<const uint32_t*>(out.ranks.back()->ptr); }
      E.cols[k].out_off = off; off += 1 + E.cols[k].enc_bytes;
    }
    E.key_bytes = off;
    out.key_bytes = off;
    out.keys = dev_alloc(ctx, (size_t)n * off);
    out.bits = dev_alloc_zero(ctx, (size_t)off * 8);
    E.keys = static_cast<uint8_t*>(out.keys->ptr);
    E.bits = static_cast<uint32_t*>(out.bits->ptr);
    SG_CUDA(launch_sort_encode(E, ctx->stream));
    m.kernel_launches += 1;
    return out;
  }

  BatchPtr take_rows(const BatchPtr& all, const Schema& sch, const int64_t* idx, int64_t take) {
    auto out = std::make_shared<DevBatch>();
    out->rows = take;
    JoinOp helper; helper.ctx = ctx;
    for (size_t i = 0; i < sch.size(); ++i) out->cols.push_back(helper.gather_column(all->cols[i], sch[i], idx, take, false));
    m.kernel_launches += sch.size();
    return out;
  }

  // full sort: LSD radix over the encoded keys (stable), then one gather per column.  Up to SMALL_SORT_ROWS rows are ranked
  // by one CTA straight from the key columns, without an encoding and without reading anything back.  Nothing here waits for
  // the device: every temporary is released in stream order (device.hpp, size-class cache).
  BatchPtr sort_rows(const BatchPtr& all, const Schema& sch, const std::vector<Key>& ks, int64_t limit) {
    const int64_t n = all->rows;
    if (n == 0) return all;
    SG_CHECK(n < (1ll << 32), SAILGPU_ERR_UNSUPPORTED, "sort of more than 2^32 rows in one partition");
    const int64_t take = limit >= 0 ? std::min<int64_t>(limit, n) : n;
    if (n <= SMALL_SORT_ROWS) {
      const SortEncodeParams E = describe_keys(all, sch, ks);
      BufPtr order = dev_alloc(ctx, (size_t)n * 4), idx = dev_alloc(ctx, (size_t)take * 8);
      SG_CUDA(launch_small_sort_cols(E, static_cast<uint32_t*>(order->ptr), ctx->stream));
      SG_CUDA(launch_widen_u32(static_cast<const uint32_t*>(order->ptr), static_cast<int64_t*>(idx->ptr), take, ctx->stream));
      m.kernel_launches += 2;
      return take_rows(all, sch, static_cast<const int64_t*>(idx->ptr), take);
    }
    Encoded enc = encode_keys(all, sch, ks);
    std::vector<BufPtr> hold;
    const RadixScratch S = radix_scratch(ctx, n, hold);
    int sort_launches = 0;
    SG_CUDA(radix_sort_indices(static_cast<const uint8_t*>(enc.keys->ptr), enc.key_bytes, n, S, static_cast<const uint32_t*>(enc.bits->ptr), ctx->stream, &sort_launches));
    m.kernel_launches += (uint64_t)(sort_launches + 1);
    BufPtr idx = dev_alloc(ctx, (size_t)take * 8);
    SG_CUDA(launch_widen_u32(S.idx_a, static_cast<int64_t*>(idx->ptr), take, ctx->stream));
    return take_rows(all, sch, static_cast<const int64_t*>(idx->ptr), take);
  }

  // TopK: radix-select the rows that can be among the first `k` on a word that holds the leading 8 bytes of the encoded key,
  // a string key's leading bytes in place of its rank (one 8 B/row pass per 11 bits), then sort only those.  The candidates
  // carry their row number as a last key, so ties come out in input order exactly as the (stable) full sort would deliver them.
  // Returns null when the selection does not narrow the input enough.
  static constexpr int64_t TOPK_MIN_ROWS = 1 << 18, TOPK_MAX_K = 1 << 16;
  BatchPtr topk_rows(const BatchPtr& all, const Schema& sch, const std::vector<Key>& ks, int64_t k) {
    const int64_t n = all->rows;
    const SortEncodeParams E = describe_keys(all, sch, ks);
    int word_bytes = 0;         // bytes of the word that are not constant zero: nothing follows a string key
    for (int i = 0; i < E.n_keys && word_bytes < 8; ++i) word_bytes += E.cols[i].kind == SORT_VIEW ? 8 : 1 + E.cols[i].enc_bytes;
    const int total_bits = std::min(64, word_bytes * 8);
    BufPtr words = dev_alloc(ctx, (size_t)n * 8);
    const uint64_t* kp = static_cast<const uint64_t*>(words->ptr);
    SG_CUDA(launch_topk_words(E, static_cast<uint64_t*>(words->ptr), ctx->stream));
    m.kernel_launches += 1;
    const int64_t want_at_most = std::max<int64_t>(4 * k, 1 << 16);
    BufPtr hist = dev_alloc(ctx, 2048 * 4);
    std::vector<uint32_t> h(2048);
    int used = 0;
    uint64_t prefix = 0;
    int64_t below = 0, cand = n;       // rows strictly before the threshold path / rows on it
    while (used < total_bits && below + cand > want_at_most) {
      const int db = std::min(11, total_bits - used);
      SG_CUDA(cudaMemsetAsync(hist->ptr, 0, 2048 * 4, ctx->stream));
      SG_CUDA(launch_topk_hist(kp, n, used, prefix, db, static_cast<uint32_t*>(hist->ptr), ctx->stream));
      SG_CUDA(cudaMemcpyAsync(h.data(), hist->ptr, 2048 * 4, cudaMemcpyDeviceToHost, ctx->stream));
      stream_sync(ctx);
      m.kernel_launches += 1;
      int64_t run = below;
      int bin = 0;
      for (; bin < (1 << db); ++bin) { if (run + h[(size_t)bin] >= k) break; run += h[(size_t)bin]; }
      if (bin == (1 << db)) bin = (1 << db) - 1;      // k exceeds the row count: everything qualifies
      below = run; cand = h[(size_t)bin];
      prefix = (prefix << db) | (uint64_t)bin;
      used += db;
    }
    if (below + cand > std::max<int64_t>(want_at_most, n / 4)) return nullptr;       // heavy ties on the leading bytes: sort everything
    BufPtr idx = dev_alloc(ctx, (size_t)(below + cand) * 8), ctr = dev_alloc_zero(ctx, 8);
    SG_CUDA(launch_topk_compact(kp, n, used, prefix, static_cast<int64_t*>(idx->ptr), static_cast<unsigned long long*>(ctr->ptr), ctx->stream));
    m.kernel_launches += 1;
    const int64_t nc = below + cand;
    BatchPtr sub = take_rows(all, sch, static_cast<const int64_t*>(idx->ptr), nc);
    DevColumn rowno; rowno.type = T(TypeId::Int64); rowno.length = nc; rowno.data = idx;
    sub->cols.push_back(rowno);
    Schema sch2 = sch;
    sch2.push_back({"__row", T(TypeId::Int64), false});
    std::vector<Key> ks2 = ks;
    auto re = std::make_shared<Expr>(); re->kind = Expr::Col; re->col = (int)sch.size(); re->type = T(TypeId::Int64); re->nullable = false;
    ks2.push_back({re, true, true});
    BatchPtr sorted = sort_rows(sub, sch2, ks2, k);
    sorted->cols.pop_back();
    return sorted;
  }

  BatchPtr run() {
    const Schema& sch = in_schemas[0];
    BatchPtr all = concat_batches(ctx, sch, parts);
    parts.clear();
    const int64_t n = all->rows;
    if (n == 0) return all;
    SG_CHECK(n < (1ll << 32), SAILGPU_ERR_UNSUPPORTED, "sort of more than 2^32 rows in one partition");
    const char* tk = getenv("SAILGPU_TOPK_MIN_ROWS");       // tests lower it
    const int64_t topk_min = tk && *tk ? atoll(tk) : TOPK_MIN_ROWS;
    if (fetch >= 0 && fetch <= TOPK_MAX_K && n >= topk_min && 8 * fetch < n) {
      BatchPtr t = topk_rows(all, sch, keys, fetch);
      if (t) return t;
    }
    return sort_rows(all, sch, keys, fetch);
  }
};

// ================================================================================================
// SortPreservingMergeExec: k-way merge of sorted runs.  Inputs = the sorted partitions (every input is one run, its
// batches arrive in order); with "runs":"batches" every pushed batch is a run of its own (what an exchange that gathers
// the locally sorted partitions of the ranks delivers).  Output = one sorted stream, optionally the first `fetch` rows.
// ================================================================================================
struct MergeOp : SortOp {
  bool runs_are_batches = false;
  std::vector<std::vector<BatchPtr>> per_input;
  std::vector<bool> done_in;

  void push(int input, const BatchPtr& b) override {
    SG_CHECK(input >= 0 && input < (int)per_input.size(), SAILGPU_ERR_INVALID, "merge input index out of range");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    if (b->rows) per_input[(size_t)input].push_back(b);
  }
  void finish(int input) override {
    SG_CHECK(input >= 0 && input < (int)done_in.size(), SAILGPU_ERR_INVALID, "merge input index out of range");
    done_in[(size_t)input] = true;
    input_done = true;
    for (bool d : done_in) input_done = input_done && d;
  }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (!input_done) return true;
    if (emitted) return false;
    const uint64_t t0 = now_ns();
    *out = merge();
    emitted = true;
    m.elapsed_compute_ns += now_ns() - t0;
    m.output_rows += (uint64_t)(*out)->rows; m.output_batches++;
    return false;
  }

  BatchPtr merge() {
    const Schema& sch = in_schemas[0];
    std::vector<BatchPtr> runs;
    for (auto& in : per_input) {
      if (in.empty()) continue;
      if (runs_are_batches) for (auto& b : in) runs.push_back(b);
      else runs.push_back(in.size() == 1 ? in[0] : concat_batches(ctx, sch, in));
    }
    per_input.clear();
    if (runs.empty()) return empty_batch(ctx, sch);
    // with a fetch only the first `fetch` rows of every run can reach the output
    if (fetch >= 0)
      for (auto& r : runs)
        if (r->rows > fetch) {
          BufPtr idx = dev_alloc(ctx, (size_t)fetch * 8);
          SG_CUDA(launch_iota(static_cast<int64_t*>(idx->ptr), fetch, ctx->stream));
          r = take_rows(r, sch, static_cast<const int64_t*>(idx->ptr), fetch);
          stream_sync(ctx);
        }
    if (runs.size() == 1) return runs[0];
    std::vector<int64_t> off(runs.size() + 1, 0);
    for (size_t i = 0; i < runs.size(); ++i) off[i + 1] = off[i] + runs[i]->rows;
    BatchPtr all = concat_batches(ctx, sch, runs);
    const int64_t n = all->rows;
    Encoded enc = encode_keys(all, sch, keys);
    BufPtr doff = dev_alloc(ctx, off.size() * 8), perm = dev_alloc(ctx, (size_t)n * 8);
    SG_CUDA(cudaMemcpyAsync(doff->ptr, off.data(), off.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    SG_CUDA(launch_merge_rank(static_cast<const uint8_t*>(enc.keys->ptr), enc.key_bytes, static_cast<const int64_t*>(doff->ptr), (int)runs.size(), n,
                              static_cast<int64_t*>(perm->ptr), ctx->stream));
    m.kernel_launches += 1;
    const int64_t take = fetch >= 0 ? std::min<int64_t>(fetch, n) : n;
    BatchPtr out = take_rows(all, sch, static_cast<const int64_t*>(perm->ptr), take);
    stream_sync(ctx);       // `off` is a host vector
    return out;
  }
};

static void parse_sort_keys(SortOp* op, const Json& spec, const Schema& in) {
  for (auto& k : spec.at("keys").a) {
    SortOp::Key key;
    key.e = parse_expr(k.at("expr"), in);
    const Json* asc = k.find("asc"); key.asc = !asc || asc->kind != Json::Bool || asc->b;
    const Json* nf = k.find("nulls_first"); key.nulls_first = nf && nf->kind == Json::Bool ? nf->b : key.asc;
    op->keys.push_back(key);
  }
  SG_CHECK(!op->keys.empty() && op->keys.size() <= 7, SAILGPU_ERR_INVALID, "sort needs 1..7 keys");
  for (auto& k : op->keys) {      // plan-time limits (sailgpu_spec_validate)
    SG_CHECK(k.e->kind == Expr::Col, SAILGPU_ERR_UNSUPPORTED, "sort keys must be column references");
    SG_CHECK(k.e->type.id != TypeId::Float32, SAILGPU_ERR_UNSUPPORTED, "Float32 sort keys");
  }
  const Json* f = spec.find("fetch");
  if (f && !f->is_null()) op->fetch = f->as_int();
}

std::unique_ptr<Op> make_merge_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs) {
  SG_CHECK(!inputs.empty(), SAILGPU_ERR_INVALID, "sort_preserving_merge takes one input per sorted partition");
  for (auto& s : inputs) {
    SG_CHECK(s.size() == inputs[0].size(), SAILGPU_ERR_INVALID, "sort_preserving_merge inputs differ in schema");
    for (size_t i = 0; i < s.size(); ++i) SG_CHECK(s[i].type == inputs[0][i].type, SAILGPU_ERR_INVALID, "sort_preserving_merge inputs differ in schema");
  }
  auto op = std::make_unique<MergeOp>();
  op->ctx = ctx; op->kind = "sort_preserving_merge"; op->in_schemas = inputs; op->out_schema = inputs[0];
  parse_sort_keys(op.get(), spec, inputs[0]);
  const Json* r = spec.find("runs");
  op->runs_are_batches = r && !r->is_null() && r->as_str() == "batches";
  op->per_input.resize(inputs.size());
  op->done_in.assign(inputs.size(), false);
  return op;
}

std::unique_ptr<Op> make_sort_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs) {
  SG_CHECK(inputs.size() == 1, SAILGPU_ERR_INVALID, "sort takes one input");
  auto op = std::make_unique<SortOp>();
  op->ctx = ctx; op->kind = "sort"; op->in_schemas = inputs; op->out_schema = inputs[0];
  parse_sort_keys(op.get(), spec, inputs[0]);
  return op;
}

// ================================================================================================
// AggregateExec whose group key does not fit the hash table (more than 6 keys or more than 64 packed key bytes; TPC-H Q10
// groups by seven columns, four of them strings): grouping by SORTING.  The key expressions are evaluated as columns, encoded
// with the sort operator's order-preserving encoding and radix-sorted; runs of equal keys get dense group numbers; the
// aggregate itself then runs through the ordinary hash pipeline on that ONE Int64 key; the key columns of the result are
// gathered from one representative row per group.  DataFusion's GroupValuesRows handles such keys in its row format
// (datafusion physical-plan aggregates/group_values) -- same result rows, unspecified order.
// ================================================================================================
std::unique_ptr<Op> make_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs, int partition);

struct WideAggOp : Op {
  Json spec;
  std::vector<BatchPtr> parts;
  bool input_done = false, emitted = false;
  int n_keys = 0;
  bool merging = false, partial = false;

  static Json jnum(int64_t v) { Json j; j.kind = Json::Num; j.s = std::to_string(v); return j; }
  static Json jstr(const std::string& v) { Json j; j.kind = Json::Str; j.s = v; return j; }
  static Json jobj(std::vector<std::pair<std::string, Json>> v) { Json j; j.kind = Json::Obj; j.o = std::move(v); return j; }
  static Json jarr(std::vector<Json> v) { Json j; j.kind = Json::Arr; j.a = std::move(v); return j; }
  static Json jcol(int64_t i) { return jobj({{"col", jnum(i)}}); }

  void push(int input, const BatchPtr& b) override {
    SG_CHECK(input == 0, SAILGPU_ERR_INVALID, "aggregate has one input");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    if (b->rows) parts.push_back(b);
  }
  void finish(int) override { input_done = true; }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (!input_done) return true;
    if (emitted) return false;
    const uint64_t t0 = now_ns();
    *out = run();
    emitted = true;
    m.elapsed_compute_ns += now_ns() - t0;
    m.output_rows += (uint64_t)(*out)->rows; m.output_batches++;
    return false;
  }

  BatchPtr through(const Json& sub_spec, const Schema& in, const BatchPtr& b, Schema* out_schema) {
    std::unique_ptr<Op> op = make_op(ctx, sub_spec, {in}, 0);
    if (b->rows) op->push(0, b);
    op->finish(0);
    std::vector<BatchPtr> outs;
    for (;;) { BatchPtr o; const bool more = op->pull(&o); if (o && o->rows) outs.push_back(o); if (!more) break; }
    m.kernel_launches += op->m.kernel_launches;
    if (out_schema) *out_schema = op->out_schema;
    return outs.empty() ? empty_batch(ctx, op->out_schema) : outs.size() == 1 ? outs[0] : concat_batches(ctx, op->out_schema, outs);
  }

  BatchPtr run() {
    const Schema& in = in_schemas[0];
    if (parts.empty()) return empty_batch(ctx, out_schema);
    BatchPtr all = parts.size() == 1 ? parts[0] : concat_batches(ctx, in, parts);
    parts.clear();
    const int64_t n = all->rows;
    SG_CHECK(n < (1ll << 32), SAILGPU_ERR_UNSUPPORTED, "sort-based grouping of more than 2^32 rows in one partition");
    // 1. the group expressions as columns
    const Json& gb = spec.at("group_by");
    std::vector<Json> kex;
    for (size_t i = 0; i < gb.a.size(); ++i) kex.push_back(jobj({{"expr", gb.a[i].at("expr")}, {"name", jstr("__k" + std::to_string(i))}}));
    Schema ks;
    BatchPtr kb = through(jobj({{"op", jstr("projection")}, {"exprs", jarr(kex)}}), in, all, &ks);
    // 2. rows with equal keys next to each other: ordered by a 64-bit hash of the key columns (8 radix digits whatever the key
    //    width); only if two different keys share a hash -- equal keys would then not be adjacent -- by the sort encoding
    SortOp so; so.ctx = ctx;
    std::vector<SortOp::Key> keys;
    for (int i = 0; i < n_keys; ++i) keys.push_back({parse_expr(jcol(i), ks), true, true});
    const SortEncodeParams E = so.describe_keys(kb, ks, keys);
    std::vector<BufPtr> hold;
    const RadixScratch S = radix_scratch(ctx, n, hold);
    int sort_launches = 0;
    BufPtr hk = dev_alloc(ctx, (size_t)n * 8), all_bits = dev_alloc(ctx, 16 * 4), coll = dev_alloc_zero(ctx, 8);
    SG_CUDA(cudaMemsetAsync(all_bits->ptr, 0xFF, 16 * 4, ctx->stream));
    SG_CUDA(launch_group_hash(E, static_cast<uint8_t*>(hk->ptr), ctx->stream));
    SG_CUDA(radix_sort_indices(static_cast<const uint8_t*>(hk->ptr), 8, n, S, static_cast<const uint32_t*>(all_bits->ptr), ctx->stream, &sort_launches));
    // 3. runs of equal keys -> dense group numbers, one representative row per group
    BufPtr heads = dev_alloc(ctx, (size_t)n * 4), before = dev_alloc(ctx, (size_t)n * 8), scr2 = dev_alloc(ctx, 1026 * 8);
    SG_CUDA(launch_group_heads(E, S.idx_a, static_cast<uint32_t*>(heads->ptr), static_cast<const uint8_t*>(hk->ptr), static_cast<unsigned long long*>(coll->ptr),
                               ctx->stream));
    unsigned long long n_coll = 0;
    SG_CUDA(cudaMemcpyAsync(&n_coll, coll->ptr, 8, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    if (n_coll != 0 || getenv("SAILGPU_WIDEAGG_FULL_SORT") != nullptr) {
      int more = 0;
      SortOp::Encoded enc = so.encode_keys(kb, ks, keys);
      SG_CUDA(radix_sort_indices(static_cast<const uint8_t*>(enc.keys->ptr), enc.key_bytes, n, S, static_cast<const uint32_t*>(enc.bits->ptr), ctx->stream, &more));
      SG_CUDA(launch_group_heads(E, S.idx_a, static_cast<uint32_t*>(heads->ptr), nullptr, nullptr, ctx->stream));
      sort_launches += more + 1 + (int)so.m.kernel_launches;
    }
    SG_CUDA(launch_exclusive_scan_u32(static_cast<const uint32_t*>(heads->ptr), n, static_cast<uint64_t*>(before->ptr), static_cast<uint64_t*>(scr2->ptr), ctx->stream));
    uint64_t n_groups = 0;
    SG_CUDA(cudaMemcpyAsync(&n_groups, static_cast<uint64_t*>(scr2->ptr) + std::min<int64_t>(1024, (n + 4095) / 4096), 8, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    DevColumn gid; gid.type = T(TypeId::Int64); gid.length = n; gid.data = dev_alloc(ctx, (size_t)n * 8);
    BufPtr rep = dev_alloc(ctx, (size_t)n_groups * 8);
    SG_CUDA(launch_assign_groups(S.idx_a, static_cast<const uint32_t*>(heads->ptr), static_cast<const uint64_t*>(before->ptr), n,
                                 static_cast<int64_t*>(gid.data->ptr), static_cast<int64_t*>(rep->ptr), ctx->stream));
    m.kernel_launches += (uint64_t)sort_launches + 4;
    // 4. the aggregate on the group number.  Merging modes find their state columns by position (after the keys): [gid | states];
    //    the others address input columns by index: [inputs | gid]
    auto agg_in = std::make_shared<DevBatch>();
    agg_in->rows = n;
    Schema ain;
    Field gf; gf.name = "__gid"; gf.type = T(TypeId::Int64); gf.nullable = false;
    int gid_col = 0;
    if (merging) {
      ain.push_back(gf); agg_in->cols.push_back(gid);
      for (size_t i = (size_t)n_keys; i < in.size(); ++i) { ain.push_back(in[i]); agg_in->cols.push_back(all->cols[i]); }
    } else {
      ain = in; agg_in->cols = all->cols;
      gid_col = (int)in.size();
      ain.push_back(gf); agg_in->cols.push_back(gid);
    }
    std::vector<std::pair<std::string, Json>> so2;
    for (auto& kv : spec.o) {
      if (kv.first == "group_by") so2.push_back({"group_by", jarr({jobj({{"expr", jcol(gid_col)}, {"name", jstr("__gid")}})})});
      else so2.push_back(kv);
    }
    Schema aos;
    BatchPtr agg = through(jobj(so2), ain, agg_in, &aos);
    // a partial aggregate in partitioned mode may emit a group more than once
    SG_CHECK((uint64_t)agg->rows == n_groups || (partial && (uint64_t)agg->rows > n_groups), SAILGPU_ERR_STATE, "sort-based grouping: group count mismatch");
    // 5. key columns of the result: the representative row of each output group
    JoinOp helper; helper.ctx = ctx;
    DevColumn repc; repc.type = T(TypeId::Int64); repc.length = (int64_t)n_groups; repc.data = rep;
    DevColumn pick = helper.gather_column(repc, gf, static_cast<const int64_t*>(agg->cols[0].data->ptr), agg->rows, false);
    auto out = std::make_shared<DevBatch>();
    out->rows = agg->rows;
    for (int i = 0; i < n_keys; ++i) {
      DevColumn c = helper.gather_column(kb->cols[(size_t)i], ks[(size_t)i], static_cast<const int64_t*>(pick.data->ptr), agg->rows, false);
      out->cols.push_back(c);
    }
    for (size_t i = 1; i < agg->cols.size(); ++i) out->cols.push_back(agg->cols[i]);
    m.kernel_launches += (uint64_t)n_keys + 1;
    stream_sync(ctx);
    return out;
  }
};

std::unique_ptr<Op> make_wide_agg_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs, const Schema& out_schema) {
  auto op = std::make_unique<WideAggOp>();
  op->ctx = ctx; op->kind = "aggregate"; op->in_schemas = inputs; op->out_schema = out_schema; op->spec = spec;
  op->n_keys = (int)spec.at("group_by").a.size();
  const std::string mode = spec.at("mode").as_str();
  op->merging = mode == "final" || mode == "final_partitioned";
  op->partial = mode == "partial";
  SG_CHECK(op->n_keys >= 1 && op->n_keys <= 7, SAILGPU_ERR_UNSUPPORTED, "sort-based grouping takes 1 to 7 group keys");
  for (int i = 0; i < op->n_keys; ++i) {
    const DataType& t = out_schema[(size_t)i].type;
    SG_CHECK(t.id != TypeId::Float32, SAILGPU_ERR_UNSUPPORTED, "Float32 group keys");
  }
  return op;
}

// ================================================================================================
// RepartitionExec Hash(exprs, n): histogram -> offsets -> scatter (two passes of SINK_PARTITION)
// ================================================================================================
struct RepartitionOp : Op {
  int n_parts = 1;
  std::vector<ExprPtr> exprs;
  PipelineRunner run;
  std::vector<std::deque<BatchPtr>> ready;     // per partition
  bool input_done = false;
  int rr = 0;
  // RowRoundRobinPartitioner (crates/sail-physical-plan/src/repartition.rs:46-84): row i of the running stream goes to
  // partition (next_idx + i) % n, next_idx seeded with (input_partition * n) / num_input_partitions
  bool row_round_robin = false;
  int64_t next_idx = 0;

  void partition_round_robin(const BatchPtr& b) {
    const int64_t n = b->rows;
    JoinOp helper; helper.ctx = ctx;
    for (int p = 0; p < n_parts; ++p) {
      const int64_t first = ((int64_t)p - next_idx % n_parts + n_parts) % n_parts;      // first row of this batch that lands in p
      if (first >= n) continue;
      const int64_t k = (n - first + n_parts - 1) / n_parts;
      BufPtr idx = dev_alloc(ctx, (size_t)k * 8);
      SG_CUDA(launch_iota_stride(static_cast<int64_t*>(idx->ptr), first, n_parts, k, ctx->stream));
      auto pb = std::make_shared<DevBatch>();
      pb->rows = k;
      for (size_t c = 0; c < b->cols.size(); ++c) pb->cols.push_back(helper.gather_column(b->cols[c], in_schemas[0][c], static_cast<const int64_t*>(idx->ptr), k, false));
      m.kernel_launches += 1 + b->cols.size();
      ready[(size_t)p].push_back(pb);
    }
    next_idx = (next_idx + n) % n_parts;
    stream_sync(ctx);       // the index vectors are released on return
  }

  void push(int input, const BatchPtr& b) override {
    SG_CHECK(input == 0, SAILGPU_ERR_INVALID, "repartition has one input");
    const uint64_t t0 = now_ns();
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    if (b->rows && row_round_robin) partition_round_robin(b);
    else if (b->rows) partition(b);
    m.elapsed_compute_ns += now_ns() - t0;
  }
  void finish(int) override { input_done = true; }
  bool pull(BatchPtr* out) override {      // partitions in round-robin order
    *out = nullptr;
    for (int t = 0; t < n_parts; ++t) {
      const int p = (rr + t) % n_parts;
      if (!ready[(size_t)p].empty()) { *out = ready[(size_t)p].front(); ready[(size_t)p].pop_front(); rr = p + 1; break; }
    }
    bool any = false; for (auto& q : ready) any |= !q.empty();
    if (*out) { m.output_rows += (uint64_t)(*out)->rows; m.output_batches++; }
    return any || !input_done;
  }
  bool pull_partition(int p, BatchPtr* out) override {
    SG_CHECK(p >= 0 && p < n_parts, SAILGPU_ERR_INVALID, "partition index out of range");
    *out = nullptr;
    if (!ready[(size_t)p].empty()) { *out = ready[(size_t)p].front(); ready[(size_t)p].pop_front(); m.output_rows += (uint64_t)(*out)->rows; m.output_batches++; }
    return !ready[(size_t)p].empty() || !input_done;
  }

  void partition(const BatchPtr& b) {
    auto cp = run.compiled_for(*b);
    const int64_t n = b->rows;
    BufPtr counts = dev_alloc_zero(ctx, (size_t)n_parts * 8), offsets = dev_alloc(ctx, (size_t)n_parts * 8);
    PipelineAux aux; memset(&aux, 0, sizeof(aux));
    aux.part.n_parts = n_parts;
    aux.part.n_keys = (int)cp->keys.size();
    for (size_t i = 0; i < cp->keys.size(); ++i) aux.part.keys[i] = cp->keys[i];
    aux.part.part_counts = static_cast<unsigned long long*>(counts->ptr);
    aux.part.part_offsets = static_cast<const int64_t*>(offsets->ptr);
    aux.part.pid_slot = NO_SLOT;
    aux.part.smem_off = cp->scratch_off;
    // pass 0: histogram
    PipelineParams P;
    run.prepare(P, *cp, *b, 0, n);
    P.n_out = 0;
    aux.part.pass = 0;
    run.launch(P, cp, &aux, m);
    std::vector<int64_t> cnt((size_t)n_parts), off((size_t)n_parts);
    SG_CUDA(cudaMemcpyAsync(cnt.data(), counts->ptr, (size_t)n_parts * 8, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    int64_t run_off = 0;
    for (int p = 0; p < n_parts; ++p) { off[(size_t)p] = run_off; run_off += cnt[(size_t)p]; }
    SG_CUDA(cudaMemcpyAsync(offsets->ptr, off.data(), (size_t)n_parts * 8, cudaMemcpyHostToDevice, ctx->stream));
    SG_CUDA(cudaMemsetAsync(counts->ptr, 0, (size_t)n_parts * 8, ctx->stream));
    // pass 1: scatter into one buffer per column, partition p at [off[p], off[p]+cnt[p])
    run.prepare(P, *cp, *b, 0, n);
    P.n_out = (int)cp->outs.size();
    std::vector<DevColumn> cols;
    std::vector<BufPtr> vbytes((size_t)P.n_out), bbytes((size_t)P.n_out);
    std::vector<BufPtr> heaps;
    for (auto& c : b->cols) if (c.type.is_string()) for (auto& h : c.heaps) heaps.push_back(h);
    for (int j = 0; j < P.n_out; ++j) {
      OutputCol o = cp->outs[(size_t)j];
      DevColumn c; c.type = cp->out_types[(size_t)j]; c.arrow_is_utf8 = c.type.id == TypeId::Utf8;
      if (o.width) { c.data = dev_alloc(ctx, (size_t)n * o.width); o.data = static_cast<uint8_t*>(c.data->ptr); }
      else { bbytes[(size_t)j] = dev_alloc(ctx, (size_t)n + 4); o.data = static_cast<uint8_t*>(bbytes[(size_t)j]->ptr); }
      if (o.valid_slot != NO_SLOT) { vbytes[(size_t)j] = dev_alloc(ctx, (size_t)n + 4); o.valid_bytes = static_cast<uint8_t*>(vbytes[(size_t)j]->ptr); }
      if (c.type.is_string()) c.heaps = heaps;
      P.out[j] = o;
      cols.push_back(c);
    }
    aux.part.pass = 1;
    run.launch(P, cp, &aux, m);
    check_device_error(ctx, run.scal.error());
    // slice per partition (byte columns are re-packed per partition so every bitmap starts at bit 0)
    for (int p = 0; p < n_parts; ++p) {
      const int64_t o = off[(size_t)p], k = cnt[(size_t)p];
      if (k == 0) continue;
      auto pb = std::make_shared<DevBatch>();
      pb->rows = k;
      for (int j = 0; j < P.n_out; ++j) {
        DevColumn c = cols[(size_t)j];
        c.length = k;
        if (bbytes[(size_t)j]) {
          c.data = dev_alloc_zero(ctx, (size_t)((k + 31) / 32 * 4));
          SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(bbytes[(size_t)j]->ptr) + o, static_cast<uint32_t*>(c.data->ptr), k, nullptr, ctx->stream));
        } else {
          auto view = std::make_shared<DevBuf>();
          const int w = c.type.is_string() ? 16 : c.type.arrow_width();
          view->ptr = static_cast<uint8_t*>(cols[(size_t)j].data->ptr) + o * w; view->bytes = (size_t)k * w;
          BufPtr keep = cols[(size_t)j].data;
          view->on_release = [keep] {};
          c.data = view;
        }
        if (vbytes[(size_t)j]) {
          c.validity = dev_alloc_zero(ctx, (size_t)((k + 31) / 32 * 4));
          SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(vbytes[(size_t)j]->ptr) + o, static_cast<uint32_t*>(c.validity->ptr), k, nullptr, ctx->stream));
          c.null_count = -1;
        }
        pb->cols.push_back(c);
      }
      ready[(size_t)p].push_back(pb);
    }
    stream_sync(ctx);
  }
};

std::unique_ptr<Op> make_repartition_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs) {
  SG_CHECK(inputs.size() == 1, SAILGPU_ERR_INVALID, "repartition takes one input");
  auto op = std::make_unique<RepartitionOp>();
  op->ctx = ctx; op->kind = "repartition"; op->in_schemas = inputs; op->out_schema = inputs[0];
  const Json* sch = spec.find("scheme");
  const std::string scheme = sch ? sch->as_str() : "hash";
  SG_CHECK(scheme == "hash" || scheme == "round_robin_row", SAILGPU_ERR_UNSUPPORTED,
           "repartition scheme '" + scheme + "': Partitioning::Hash and the row round-robin of ExplicitRepartitionExec run on the GPU; "
           "RoundRobinBatch only re-labels whole batches and stays with the reference's stream plumbing (SURVEY.md 8b)");
  op->n_parts = (int)spec.at("n").as_int();
  SG_CHECK(op->n_parts >= 1 && op->n_parts <= 4096, SAILGPU_ERR_INVALID, "partition count out of range");
  if (scheme == "round_robin_row") {
    const Json* ip = spec.find("input_partition"); const Json* np = spec.find("num_input_partitions");
    const int64_t in_part = ip && !ip->is_null() ? ip->as_int() : 0, n_in = np && !np->is_null() ? np->as_int() : 1;
    SG_CHECK(n_in >= 1 && in_part >= 0 && in_part < n_in, SAILGPU_ERR_INVALID, "input_partition / num_input_partitions out of range");
    op->row_round_robin = true;
    op->next_idx = (in_part * op->n_parts) / n_in;
    op->ready.resize((size_t)op->n_parts);
    return op;
  }
  for (auto& e : spec.at("exprs").a) op->exprs.push_back(parse_expr(e, inputs[0]));
  SG_CHECK(!op->exprs.empty() && (int)op->exprs.size() <= MAX_KEYS, SAILGPU_ERR_INVALID, "hash repartition needs 1.." + std::to_string(MAX_KEYS) + " key expressions");
  op->ready.resize((size_t)op->n_parts);
  op->run.init(ctx, inputs[0]);
  auto* raw = op.get();
  op->run.custom_sink = [raw](PipelineCompiler& pc, CompiledPipeline& cp) {
    pc.finish_partition(cp, raw->exprs);
    cp.extra_scratch = (uint32_t)(raw->n_parts * 16 + 16);      // u32 cnt[n] + u64 base[n] per CTA
  };
  return op;
}


// ================================================================================================
// ExchangeOp -- the shuffle boundary as an operator, so that a whole two-phase aggregation
//   [partial] -> exchange(auto) -> [final] -> exchange(gather) -> [sort]
// runs as ONE chain inside the library: no host round trip, no Arrow export/import between the stages.
//   mode "hash":   RepartitionExec Hash(exprs, world) + all-to-all (partition p -> rank p)
//   mode "gather": everything to rank `root` (CoalescePartitionsExec / InputMode::Merge)
//   mode "auto":   hash, unless every rank holds at most `small_rows` rows -- then gather (a handful of partial rows per
//                  rank, TPC-H Q1: hashing them costs a second exchange for nothing).  The choice is taken on an
//                  all-gather of the row counts, so every rank takes the same one; a later "gather" exchange of the same
//                  chain sees that the rows already sit on the root and does not communicate.
// ================================================================================================
BatchPtr exchange_batches(Ctx* ctx, const Schema& schema, const std::vector<BatchPtr>& parts, std::vector<int64_t>* source_offsets = nullptr, int64_t abort_above_rows = -1);
std::unique_ptr<Op> make_repartition_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs);

struct ExchangeOp : Op {
  std::string mode = "gather";
  int root = 0;
  int64_t small_rows = 1 << 14;
  Json exprs_json;
  std::vector<BatchPtr> parts_in;
  BatchPtr result;
  bool done = false, pulled = false;
  bool* on_root_hint = nullptr;     // shared by the exchanges of one chain (owned by the ChainOp)
  bool keep_runs = false;           // emit what every source rank sent as a batch of its own (input of a sort-preserving merge)
  std::deque<BatchPtr> run_batches;

  void split_runs(const std::vector<int64_t>& off) {
    JoinOp helper; helper.ctx = ctx;
    const Schema& sch = in_schemas[0];
    for (size_t s = 0; s + 1 < off.size(); ++s) {
      const int64_t k = off[s + 1] - off[s];
      if (k == 0) continue;
      if (k == result->rows) { run_batches.push_back(result); continue; }
      BufPtr idx = dev_alloc(ctx, (size_t)k * 8);
      SG_CUDA(launch_iota_stride(static_cast<int64_t*>(idx->ptr), off[s], 1, k, ctx->stream));
      auto b = std::make_shared<DevBatch>();
      b->rows = k;
      for (size_t c = 0; c < sch.size(); ++c) b->cols.push_back(helper.gather_column(result->cols[c], sch[c], static_cast<const int64_t*>(idx->ptr), k, false));
      stream_sync(ctx);
      run_batches.push_back(b);
    }
    if (run_batches.empty()) run_batches.push_back(result);
  }

  void push(int input, const BatchPtr& b) override {
    SG_CHECK(input == 0, SAILGPU_ERR_INVALID, "exchange has one input");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    if (b->rows) parts_in.push_back(b);
  }
  void finish(int) override {
    const uint64_t t0 = now_ns();
    const Schema& sch = in_schemas[0];
    BatchPtr all = parts_in.empty() ? empty_batch(ctx, sch) : concat_batches(ctx, sch, parts_in);
    parts_in.clear();
    const int W = ctx->world;
    if (W == 1) { result = all; done = true; if (keep_runs) run_batches.push_back(result); return; }
    std::vector<int64_t> src_off;
    if (mode == "gather" && on_root_hint && *on_root_hint) {       // an "auto" exchange of this chain already coalesced on the root
      result = all; done = true; if (keep_runs) run_batches.push_back(result); return;
    }
    std::vector<BatchPtr> parts((size_t)W);
    bool sent = false;
    if (mode == "gather" || mode == "auto") {
      // "auto" tries the coalescing layout first: the all-gathered count table of that attempt tells every rank whether some
      // rank holds more than small_rows rows -- if so nothing was sent and the rows are hash-partitioned instead
      for (int p = 0; p < W; ++p) parts[(size_t)p] = p == root ? all : empty_batch(ctx, sch);
      result = exchange_batches(ctx, sch, parts, keep_runs ? &src_off : nullptr, mode == "auto" ? small_rows : -1);
      sent = result != nullptr;
      if (on_root_hint) *on_root_hint = sent && mode == "auto";
    }
    if (!sent) {
      if (on_root_hint) *on_root_hint = false;
      Json spec; spec.kind = Json::Obj;
      Json opk; opk.kind = Json::Str; opk.s = "repartition";
      Json sc; sc.kind = Json::Str; sc.s = "hash";
      Json nn; nn.kind = Json::Num; nn.s = std::to_string(W);
      spec.o = {{"op", opk}, {"scheme", sc}, {"exprs", exprs_json}, {"n", nn}};
      auto rp = make_repartition_op(ctx, spec, {sch});
      if (all->rows) rp->push(0, all);
      rp->finish(0);
      for (int p = 0; p < W; ++p) {
        std::vector<BatchPtr> segs;
        for (;;) { BatchPtr b; const bool more = rp->pull_partition(p, &b); if (b && b->rows) segs.push_back(b); if (!more) break; }
        parts[(size_t)p] = segs.empty() ? empty_batch(ctx, sch) : segs.size() == 1 ? segs[0] : concat_batches(ctx, sch, segs);
      }
      m.kernel_launches += rp->m.kernel_launches;
      result = exchange_batches(ctx, sch, parts, keep_runs ? &src_off : nullptr);
    }
    if (keep_runs) split_runs(src_off);
    done = true;
    m.elapsed_compute_ns += now_ns() - t0;
  }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (keep_runs) {
      if (!done) return true;
      if (!run_batches.empty()) { *out = run_batches.front(); run_batches.pop_front(); m.output_rows += (uint64_t)(*out)->rows; m.output_batches++; }
      if (run_batches.empty()) { pulled = true; result.reset(); }
      return !pulled;
    }
    if (done && !pulled) { *out = result; pulled = true; m.output_rows += (uint64_t)result->rows; m.output_batches++; result.reset(); }
    return !pulled;
  }
};

std::unique_ptr<Op> make_exchange_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs) {
  SG_CHECK(inputs.size() == 1, SAILGPU_ERR_INVALID, "exchange takes one input");
  auto op = std::make_unique<ExchangeOp>();
  op->ctx = ctx; op->kind = "exchange"; op->in_schemas = inputs; op->out_schema = inputs[0];
  const Json* md = spec.find("mode");
  if (md) op->mode = md->as_str();
  SG_CHECK(op->mode == "hash" || op->mode == "gather" || op->mode == "auto", SAILGPU_ERR_INVALID, "exchange mode must be hash, gather or auto");
  const Json* rt = spec.find("root"); if (rt && !rt->is_null()) op->root = (int)rt->as_int();
  const Json* sr = spec.find("small_rows"); if (sr && !sr->is_null()) op->small_rows = sr->as_int();
  const Json* kr = spec.find("keep_runs"); op->keep_runs = kr && kr->kind == Json::Bool && kr->b;
  if (op->mode != "gather") {
    op->exprs_json = spec.at("exprs");
    for (auto& e : op->exprs_json.a) (void)parse_expr(e, inputs[0]);          // validate at plan time
  }
  return op;
}

// ================================================================================================
// A linear chain of GPU operators executed as one island: batches move between the stages as HBM
// batches inside the library (no Arrow export/import, no host round trip between stages).  This is
// what the rewrite pass emits for consecutive replaced nodes, e.g. Q1's
//   pipeline[Filter+Projection+Aggregate(Partial)] -> Aggregate(FinalPartitioned) -> Sort.
// ================================================================================================
struct ChainOp : Op {
  std::vector<std::unique_ptr<Op>> ops;
  bool finished = false;
  bool rows_on_root_only = false;   // hint passed from an "auto" exchange to a later "gather" exchange of this chain
  void pump(size_t from) {
    for (size_t i = from; i + 1 < ops.size(); ++i) {
      for (;;) {
        BatchPtr b;
        const bool more = ops[i]->pull(&b);
        if (b && b->rows >= 0 && (b->rows > 0 || !more)) ops[i + 1]->push(0, b);
        if (!b || !more) break;
      }
    }
  }
  void push(int input, const BatchPtr& b) override {
    SG_CHECK(input == 0, SAILGPU_ERR_INVALID, "chain has one input");
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    ops[0]->push(0, b);
    pump(0);
  }
  void finish(int) override {
    for (size_t i = 0; i < ops.size(); ++i) {
      ops[i]->finish(0);
      if (i + 1 < ops.size()) {
        for (;;) {
          BatchPtr b;
          const bool more = ops[i]->pull(&b);
          if (b && (b->rows > 0 || !more)) ops[i + 1]->push(0, b);
          if (!more) break;
        }
      }
    }
    finished = true;
    // gpu.pipeline_* of a chain describe its FIRST stage (the pass over the input batches: the dominant kernel);
    // every stage counts towards gpu.kernel_launches
    for (auto& o : ops) m.kernel_launches += o->m.kernel_launches;
    m.pipeline_launches += ops[0]->m.pipeline_launches;
    m.jit_launches += ops[0]->m.jit_launches;
    for (auto& p : ops[0]->m.pending) m.pending.push_back(p);
    ops[0]->m.pending.clear();
    m.pipeline_kernel_ns += ops[0]->m.pipeline_kernel_ns;
  }
  bool pull(BatchPtr* out) override {
    const bool more = ops.back()->pull(out);
    if (*out) { m.output_rows += (uint64_t)(*out)->rows; m.output_batches++; }
    return more;
  }
};

std::unique_ptr<Op> make_chain_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs) {
  SG_CHECK(inputs.size() == 1, SAILGPU_ERR_INVALID, "chain takes one input");
  auto op = std::make_unique<ChainOp>();
  op->ctx = ctx; op->kind = "chain"; op->in_schemas = inputs;
  Schema cur = inputs[0];
  for (auto& s : spec.at("ops").a) {
    SG_CHECK(s.at("op").as_str() != "hash_join" && s.at("op").as_str() != "repartition", SAILGPU_ERR_UNSUPPORTED, "chain stages must be single-input, single-output operators");
    op->ops.push_back(make_op(ctx, s, {cur}, 0));
    if (auto* x = dynamic_cast<ExchangeOp*>(op->ops.back().get())) x->on_root_hint = &op->rows_on_root_only;
    cur = op->ops.back()->out_schema;
  }
  SG_CHECK(!op->ops.empty(), SAILGPU_ERR_INVALID, "empty chain");
  op->out_schema = cur;
  return op;
}

}  // namespace sg

// ================================================================================================
// NCCL exchange (dlopen: the library loads without NCCL; the exchange fails loudly if it is absent)
// ================================================================================================
struct Id128 { char b[128]; };
namespace {
struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, /* ncclUniqueId by value: 128 bytes */ Id128, int) = nullptr;
  int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
bool load_nccl(std::string* err) {
  if (g_nccl.h) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (auto n : names) { g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (g_nccl.h) break; }
  if (!g_nccl.h) { *err = std::string("NCCL not found: ") + dlerror(); return false; }
#define LOADSYM(field, name) *(void**)(&g_nccl.field) = dlsym(g_nccl.h, name); if (!g_nccl.field) { *err = std::string("NCCL symbol missing: ") + name; return false; }
  LOADSYM(GetUniqueId, "ncclGetUniqueId") LOADSYM(CommInitRank, "ncclCommInitRank") LOADSYM(Send, "ncclSend") LOADSYM(Recv, "ncclRecv")
  LOADSYM(GroupStart, "ncclGroupStart") LOADSYM(GroupEnd, "ncclGroupEnd") LOADSYM(AllGather, "ncclAllGather") LOADSYM(GetErrorString, "ncclGetErrorString")
#undef LOADSYM
  return true;
}
constexpr int NCCL_INT8 = 0, NCCL_INT64 = 4;
}  // namespace

struct sailgpu_ctx { sg::Ctx ctx; };
namespace sg { void set_ctx_error(const std::string& m); }

#define NCCL_CALL(expr) do { int _r = (expr); if (_r != 0) sg::fail(SAILGPU_ERR_CUDA, std::string("NCCL error: ") + g_nccl.GetErrorString(_r) + " at " #expr); } while (0)

namespace sg {
// all-to-all of world_size device batches over the context's communicator: parts[p] goes to rank p; returns everything
// that was sent to this rank (rows of rank 0 first, then rank 1, ...).
//
// ONE host synchronisation per exchange: everything the ranks must agree on -- rows, string-heap bytes and "carries a validity
// buffer" per (source, destination, column) -- is assembled ON THE DEVICE (the heap sizes come out of the length scans without
// being read back), all-gathered, and read back once.  The layout of every send and receive follows from that table on every
// rank; null counts of the result are not read back (validity travels only for columns where some source has a bitmap, and the
// result then reports null_count = -1, "unknown").
// abort_above_rows >= 0: if any rank contributes more rows than that, nothing is sent and nullptr is returned on EVERY rank
// (the decision is taken on the all-gathered table) -- the "auto" exchange tries the coalescing layout first this way.
BatchPtr exchange_batches(Ctx* ctx, const Schema& schema, const std::vector<BatchPtr>& parts, std::vector<int64_t>* source_offsets, int64_t abort_above_rows) {
  const int n = (int)parts.size();
  SG_CHECK(n == ctx->world, SAILGPU_ERR_INVALID, "exchange needs one batch per rank");
  if (n == 1) { if (source_offsets) *source_offsets = {0, parts[0]->rows}; return parts[0]; }
  SG_CHECK(ctx->nccl_comm != nullptr, SAILGPU_ERR_STATE, "sailgpu_ctx_comm_init has not been called");
  const int W = n, me = ctx->rank;
  const size_t ncols = schema.size();
  const size_t rec = 1 + 2 * ncols;                   // rows | heap bytes per column | has-validity per column
  std::vector<int64_t> mine((size_t)W * rec, 0);
  // 1. length scans of every (destination, string column): the totals stay on the device
  struct Pending { int p; size_t ci; BufPtr offs, scratch; int64_t nblocks; };
  std::vector<Pending> pend;
  for (int p = 0; p < W; ++p) {
    mine[(size_t)p * rec] = parts[(size_t)p]->rows;
    for (size_t ci = 0; ci < ncols; ++ci) {
      const DevColumn& col = parts[(size_t)p]->cols[ci];
      const int64_t k = col.length;
      mine[(size_t)p * rec + 1 + ncols + ci] = (k > 0 && col.validity) ? 1 : 0;
      if (schema[ci].type.is_string() && k > 0) {
        BufPtr lens = dev_alloc(ctx, (size_t)k * 4), offs = dev_alloc(ctx, (size_t)k * 8), scratch = dev_alloc(ctx, 1026 * 8);
        SG_CUDA(launch_view_lengths(col.data->ptr, k, static_cast<uint32_t*>(lens->ptr), 0, ctx->stream));
        SG_CUDA(launch_exclusive_scan_u32(static_cast<uint32_t*>(lens->ptr), k, static_cast<uint64_t*>(offs->ptr), static_cast<uint64_t*>(scratch->ptr), ctx->stream));
        pend.push_back({p, ci, offs, scratch, std::min<int64_t>(1024, (k + 4095) / 4096)});
      }
    }
  }
  BufPtr dmine = dev_alloc(ctx, mine.size() * 8), dall = dev_alloc(ctx, mine.size() * 8 * (size_t)W);
  SG_CUDA(cudaMemcpyAsync(dmine->ptr, mine.data(), mine.size() * 8, cudaMemcpyHostToDevice, ctx->stream));     // pageable source: staged before return
  for (auto& q : pend)
    SG_CUDA(cudaMemcpyAsync(static_cast<int64_t*>(dmine->ptr) + (size_t)q.p * rec + 1 + q.ci, static_cast<uint64_t*>(q.scratch->ptr) + q.nblocks, 8,
                            cudaMemcpyDeviceToDevice, ctx->stream));
  NCCL_CALL(g_nccl.AllGather(dmine->ptr, dall->ptr, mine.size(), NCCL_INT64, ctx->nccl_comm, ctx->stream));
  std::vector<int64_t> all(mine.size() * (size_t)W);
  SG_CUDA(cudaMemcpyAsync(all.data(), dall->ptr, all.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
  stream_sync(ctx);                                                                  // the one synchronisation
  auto cnt = [&](int src, int dst, size_t field) { return all[((size_t)src * W + dst) * rec + field]; };
  if (abort_above_rows >= 0) {
    int64_t mx = 0;
    for (int s = 0; s < W; ++s) { int64_t r = 0; for (int d = 0; d < W; ++d) r += cnt(s, d, 0); mx = std::max(mx, r); }
    if (mx > abort_above_rows) return nullptr;
  }
  // validity of column ci travels to `dst` iff some source has a bitmap there
  auto vneed = [&](int dst, size_t ci) { for (int s = 0; s < W; ++s) if (cnt(s, dst, 1 + ncols + ci)) return true; return false; };
  // 2. what this rank sends: compact string heaps + Arrow-conformant views, validity as bytes where the destination expects it
  struct SendCol { BufPtr data, validity_bytes, heap; int64_t heap_bytes = 0; };
  std::vector<std::vector<SendCol>> sc((size_t)W, std::vector<SendCol>(ncols));
  for (int p = 0; p < W; ++p)
    for (size_t ci = 0; ci < ncols; ++ci) {
      const DevColumn& col = parts[(size_t)p]->cols[ci];
      SendCol& sd = sc[(size_t)p][ci];
      const int64_t k = col.length;
      if (k == 0) continue;
      if (schema[ci].type.id == TypeId::Bool) {
        sd.data = dev_alloc(ctx, (size_t)k);     // booleans travel as bytes
        SG_CUDA(launch_unpack_bits(static_cast<const uint8_t*>(col.data->ptr), static_cast<uint8_t*>(sd.data->ptr), k, 0, ctx->stream));
      } else if (!schema[ci].type.is_string()) sd.data = col.data;
      if (vneed(p, ci)) {
        sd.validity_bytes = dev_alloc(ctx, (size_t)k);
        if (col.validity) SG_CUDA(launch_unpack_bits(static_cast<const uint8_t*>(col.validity->ptr), static_cast<uint8_t*>(sd.validity_bytes->ptr), k, 0, ctx->stream));
        else SG_CUDA(cudaMemsetAsync(sd.validity_bytes->ptr, 1, (size_t)k, ctx->stream));
      }
    }
  for (auto& q : pend) {
    const DevColumn& col = parts[(size_t)q.p]->cols[q.ci];
    SendCol& sd = sc[(size_t)q.p][q.ci];
    const int64_t k = col.length;
    sd.heap_bytes = cnt(me, q.p, 1 + q.ci);
    sd.heap = dev_alloc(ctx, (size_t)sd.heap_bytes);
    sd.data = dev_alloc(ctx, (size_t)k * 16);
    SG_CUDA(cudaMemcpyAsync(sd.data->ptr, col.data->ptr, (size_t)k * 16, cudaMemcpyDeviceToDevice, ctx->stream));
    SG_CUDA(launch_views_to_arrow(sd.data->ptr, k, static_cast<uint64_t*>(q.offs->ptr), static_cast<uint8_t*>(sd.heap->ptr), ctx->stream));
  }
  // 3. receive layout: rows from rank 0, then rank 1, ...
  std::vector<int64_t> row_off((size_t)W + 1, 0);
  for (int s = 0; s < W; ++s) row_off[(size_t)s + 1] = row_off[(size_t)s] + cnt(s, me, 0);
  const int64_t total_rows = row_off[(size_t)W];
  if (source_offsets) *source_offsets = row_off;
  BatchPtr out = std::make_shared<DevBatch>();
  out->rows = total_rows;
  std::vector<BufPtr> vbytes(ncols), bbytes(ncols), datas(ncols), heaps(ncols);
  std::vector<char> vrecv(ncols, 0);
  std::vector<std::vector<int64_t>> heap_off(ncols, std::vector<int64_t>((size_t)W + 1, 0));
  auto width_of = [&](size_t ci) { const DataType& t = schema[ci].type; return t.is_string() ? 16 : t.id == TypeId::Bool ? 1 : t.arrow_width(); };
  for (size_t ci = 0; ci < ncols; ++ci) {
    const DataType& t = schema[ci].type;
    DevColumn col; col.type = t; col.length = total_rows; col.arrow_is_utf8 = t.id == TypeId::Utf8;
    datas[ci] = dev_alloc(ctx, (size_t)total_rows * width_of(ci));
    vrecv[ci] = vneed(me, ci) ? 1 : 0;
    if (vrecv[ci]) vbytes[ci] = dev_alloc(ctx, (size_t)total_rows + 4);
    if (t.is_string()) {
      for (int s = 0; s < W; ++s) heap_off[ci][(size_t)s + 1] = heap_off[ci][(size_t)s] + cnt(s, me, 1 + ci);
      heaps[ci] = dev_alloc(ctx, (size_t)heap_off[ci][(size_t)W]);
      col.heaps = {heaps[ci]};
    }
    if (t.id == TypeId::Bool) bbytes[ci] = datas[ci]; else col.data = datas[ci];
    out->cols.push_back(col);
  }
  // bytes of the message `src` sends to `dst` as the exchange metrics count them: every buffer rounded up to 16 bytes
  auto a16 = [](int64_t v) { return (v + 15) & ~(int64_t)15; };
  auto msg_bytes = [&](int src, int dst) {
    const int64_t k = cnt(src, dst, 0);
    int64_t tot = 0;
    for (size_t ci = 0; ci < ncols; ++ci) tot += a16(k * width_of(ci)) + (vneed(dst, ci) ? a16(k) : 0) + a16(cnt(src, dst, 1 + ci));
    return k ? tot : 0;
  };
  // bytes that cross NVLink (everything except the segment this rank keeps) and the device time of the grouped send/recv
  {
    uint64_t sent = 0, recvd = 0;
    for (int peer = 0; peer < W; ++peer) if (peer != me) { sent += (uint64_t)msg_bytes(me, peer); recvd += (uint64_t)msg_bytes(peer, me); }
    ctx->exch_sent_bytes += sent; ctx->exch_recv_bytes += recvd; ctx->exch_calls += 1;
  }
  cudaEvent_t xe0 = nullptr, xe1 = nullptr;
  if (timing_enabled()) { SG_CUDA(cudaEventCreate(&xe0)); SG_CUDA(cudaEventCreate(&xe1)); SG_CUDA(cudaEventRecord(xe0, ctx->stream)); }
  NCCL_CALL(g_nccl.GroupStart());
  struct GroupGuard { bool open = true; ~GroupGuard() { if (open) g_nccl.GroupEnd(); } } group_guard;     // an error below must not leave the group open
  for (int peer = 0; peer < W; ++peer) {
    const int64_t ks = parts[(size_t)peer]->rows, kr = cnt(peer, me, 0);
    for (size_t ci = 0; ci < ncols; ++ci) {
      const DataType& t = schema[ci].type;
      const int w = width_of(ci);
      const SendCol& sd = sc[(size_t)peer][ci];
      if (ks) {
        NCCL_CALL(g_nccl.Send(sd.data->ptr, (size_t)ks * w, NCCL_INT8, peer, ctx->nccl_comm, ctx->stream));
        if (sd.validity_bytes) NCCL_CALL(g_nccl.Send(sd.validity_bytes->ptr, (size_t)ks, NCCL_INT8, peer, ctx->nccl_comm, ctx->stream));
        if (t.is_string() && sd.heap_bytes) NCCL_CALL(g_nccl.Send(sd.heap->ptr, (size_t)sd.heap_bytes, NCCL_INT8, peer, ctx->nccl_comm, ctx->stream));
      }
      if (kr) {
        NCCL_CALL(g_nccl.Recv(static_cast<uint8_t*>(datas[ci]->ptr) + row_off[(size_t)peer] * w, (size_t)kr * w, NCCL_INT8, peer, ctx->nccl_comm, ctx->stream));
        if (vrecv[ci]) NCCL_CALL(g_nccl.Recv(static_cast<uint8_t*>(vbytes[ci]->ptr) + row_off[(size_t)peer], (size_t)kr, NCCL_INT8, peer, ctx->nccl_comm, ctx->stream));
        const int64_t hb = cnt(peer, me, 1 + ci);
        if (t.is_string() && hb) NCCL_CALL(g_nccl.Recv(static_cast<uint8_t*>(heaps[ci]->ptr) + heap_off[ci][(size_t)peer], (size_t)hb, NCCL_INT8, peer, ctx->nccl_comm, ctx->stream));
      }
    }
  }
  group_guard.open = false;
  NCCL_CALL(g_nccl.GroupEnd());
  if (xe1) { SG_CUDA(cudaEventRecord(xe1, ctx->stream)); ctx->exch_events.emplace_back(xe0, xe1); }      // read when metrics are asked for
  // 4. post-process (no read-back): rebase string views per source segment, pack byte columns into Arrow bitmaps
  for (size_t ci = 0; ci < ncols; ++ci) {
    DevColumn& col = out->cols[ci];
    if (schema[ci].type.is_string())
      for (int s = 0; s < W; ++s) {
        const int64_t kr = cnt(s, me, 0);
        if (kr) SG_CUDA(launch_rebase_views(static_cast<uint8_t*>(col.data->ptr) + row_off[(size_t)s] * 16, kr,
                                            reinterpret_cast<uint64_t>(col.heaps[0]->ptr) + (uint64_t)heap_off[ci][(size_t)s], ctx->stream));
      }
    if (bbytes[ci]) {
      col.data = dev_alloc_zero(ctx, (size_t)((total_rows + 31) / 32 * 4));
      SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(bbytes[ci]->ptr), static_cast<uint32_t*>(col.data->ptr), total_rows, nullptr, ctx->stream));
    }
    if (vrecv[ci] && total_rows > 0) {
      col.validity = dev_alloc_zero(ctx, (size_t)((total_rows + 31) / 32 * 4));
      SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(vbytes[ci]->ptr), static_cast<uint32_t*>(col.validity->ptr), total_rows, nullptr, ctx->stream));
      col.null_count = -1;
    } else col.null_count = 0;
  }
  // the staging buffers of this call are released stream-ordered (dev_alloc): nothing to wait for
  return out;
}

// device time of the grouped send/recv of finished exchanges -> gpu.exchange_ns (called when metrics are read)
void resolve_exchange_timing(Ctx* ctx) {
  for (auto& ev : ctx->exch_events) {
    float ms = 0.f;
    if (cudaEventSynchronize(ev.second) == cudaSuccess && cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) ctx->exch_ns += (uint64_t)((double)ms * 1e6);
    cudaEventDestroy(ev.first); cudaEventDestroy(ev.second);
  }
  ctx->exch_events.clear();
}
}  // namespace sg

extern "C" {

SAILGPU_API int32_t sailgpu_comm_unique_id(uint8_t* out128) {
  std::string err;
  if (!out128 || !load_nccl(&err)) return SAILGPU_ERR_CUDA;
  return g_nccl.GetUniqueId(out128) == 0 ? SAILGPU_OK : SAILGPU_ERR_CUDA;
}

SAILGPU_API int32_t sailgpu_ctx_comm_init(sailgpu_ctx* c, const uint8_t* unique_id128, int32_t rank, int32_t world_size) {
  try {
    SG_CHECK(c && unique_id128 && world_size >= 1 && rank >= 0 && rank < world_size, SAILGPU_ERR_INVALID, "bad comm_init arguments");
    std::string err;
    SG_CHECK(load_nccl(&err), SAILGPU_ERR_CUDA, err);
    std::lock_guard<std::recursive_mutex> lk(c->ctx.mu);
    SG_CUDA(cudaSetDevice(c->ctx.device));
    Id128 id; memcpy(id.b, unique_id128, 128);
    void* comm = nullptr;
    NCCL_CALL(g_nccl.CommInitRank(&comm, world_size, id, rank));
    c->ctx.nccl_comm = comm; c->ctx.rank = rank; c->ctx.world = world_size;
    return SAILGPU_OK;
  } catch (const sg::Error& e) { sg::set_ctx_error(e.what()); return e.code; }
  catch (const std::exception& e) { sg::set_ctx_error(std::string("internal error: ") + e.what()); return SAILGPU_ERR_CUDA; }
}

// all-to-all of n = world_size device batches: batch p goes to rank p; recv = everything sent to this rank
SAILGPU_API int32_t sailgpu_exchange(sailgpu_ctx* c, const struct ArrowSchema* schema_c, struct ArrowDeviceArray* send, int32_t n, struct ArrowDeviceArray* recv) {
  using namespace sg;
  try {
    SG_CHECK(c && schema_c && send && recv, SAILGPU_ERR_INVALID, "null argument");
    Ctx* ctx = &c->ctx;
    std::lock_guard<std::recursive_mutex> lk(ctx->mu);
    SG_CUDA(cudaSetDevice(ctx->device));
    SG_CHECK(n == ctx->world, SAILGPU_ERR_INVALID, "exchange needs one batch per rank");
    Schema schema = schema_from_arrow(schema_c);
    std::vector<BatchPtr> parts;
    for (int p = 0; p < n; ++p) {
      if (send[p].array.release == nullptr) { parts.push_back(empty_batch(ctx, schema)); continue; }   // nothing for rank p
      BatchPtr b = take_internal_batch(&send[p], ctx);
      if (!b) b = import_device_batch(ctx, schema, &send[p]);
      parts.push_back(b);
    }
    BatchPtr out = exchange_batches(ctx, schema, parts);
    export_device_batch(ctx, schema, out, recv);
    return SAILGPU_OK;
  } catch (const sg::Error& e) { sg::set_ctx_error(e.what()); return e.code; }
  catch (const std::exception& e) { sg::set_ctx_error(std::string("internal error: ") + e.what()); return SAILGPU_ERR_CUDA; }
}

}  // extern "C"
