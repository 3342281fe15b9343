// runner.hpp -- compiles a stage list into a tile pipeline and launches it; shared by every operator.
#pragma once
#include <algorithm>

#include "engine.hpp"
#include "jit.hpp"

namespace sg {

inline uint64_t now_ns() {
  return (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
// SAILGPU_TRACE=1: synchronising phase timer printed to stderr (diagnostics only)
struct Trace {
  Ctx* ctx; const char* what; uint64_t t0; bool on;
  Trace(Ctx* c, const char* w) : ctx(c), what(w), on(getenv("SAILGPU_TRACE") != nullptr) { if (on) { cudaStreamSynchronize(ctx->stream); t0 = now_ns(); } }
  ~Trace() { if (on) { cudaStreamSynchronize(ctx->stream); fprintf(stderr, "[sailgpu trace] %-28s %8.3f ms\n", what, (now_ns() - t0) / 1e6); } }
};

inline uint64_t next_pow2(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return p; }

// ------------------------------------------------------------------------------------------------
// launching one compiled pipeline over one batch
// ------------------------------------------------------------------------------------------------
struct DevProgram {
  BufPtr literals;
  std::vector<uint64_t> literal_ptrs;
};

inline bool timing_enabled() { static const bool on = getenv("SAILGPU_TIMING") != nullptr; return on; }

// SAILGPU_DUMP=1: prints every compiled pipeline (geometry, inputs, VM program, sink) to stderr
inline void dump_pipeline(const CompiledPipeline& cp) {
  static const char* names[] = {"NOP", "UNPACK_BITS", "CONST", "MOV", "CVT", "ADD", "SUB", "MUL", "DIV", "REM", "NEG", "MULW", "MUL128_64", "DIVROUND",
                                "EQ", "NE", "LT", "LE", "GT", "GE", "AND", "OR", "NOT", "ANDNOT", "SELECT", "STR_EQ_LONG", "STR_LIKE", "DATE_PART", "PROBE", "GATHER", "SUBSTR",
                                "TS_PART", "TS_TRUNC", "MUL_POW10_CHK", "CHAR_LEN", "DISTINCT_FIRST"};
  static const char* sinks[] = {"STORE", "COMPACT", "AGG", "BUILD", "PARTITION"};
  fprintf(stderr, "[sailgpu pipeline] sink=%s rows/thread=%d stages=%d smem=%zu B (temps %u, stage %u, hot %u) inputs=%zu outs=%zu%s\n",
          cp.sink >= 0 && cp.sink < 5 ? sinks[cp.sink] : "?", cp.rpt, cp.n_stages, cp.smem_bytes, cp.temps_bytes, cp.stage_bytes, cp.hot_bytes,
          cp.inputs.size(), cp.outs.size(), cp.cold_variant ? " [cold variant]" : "");
  for (auto& in : cp.inputs) fprintf(stderr, "  in  col %d%s width %u -> slot %d\n", in.col, in.validity ? " (validity)" : "", in.width, in.slot);
  for (size_t i = 0; i < cp.prog.size(); ++i) {
    const VmInst& I = cp.prog[i];
    const int base = I.op & 0xFF, kind = I.op >> 8;
    fprintf(stderr, "  %2zu  %-12s k%d dst=%d a=%d b=%d c=%d flags=%u aux=%u imm=%lld\n", i, base < OP_COUNT_ ? names[base] : "?", kind, (int)I.dst, (int)I.a, (int)I.b,
            (int)I.c, I.flags, I.aux, (long long)I.imm0);
  }
  if (cp.sink == SINK_AGG)
    fprintf(stderr, "  agg keys=%d key_words=%d accs=%d entry_words=%d hot_groups=%d reg_path=%d\n", cp.agg.n_keys, cp.agg.key_words, cp.agg.n_accs, cp.agg.entry_words,
            cp.agg.hot_groups, cp.agg.reg_path);
}

// what a runner compiles; shared between runners of identical operators (PipelineRunner::share)
struct RunnerShared {
  std::map<std::vector<bool>, std::shared_ptr<CompiledPipeline>> cache;
  std::map<const CompiledPipeline*, DevProgram> programs;
};

struct PipelineRunner {
  Ctx* ctx;
  Schema in_schema;
  std::vector<StageSpec> stages;
  std::shared_ptr<RunnerShared> shared_state = std::make_shared<RunnerShared>();
  // adopt the compiled pipelines of every earlier operator with this key on this context (plain filter / projection /
  // aggregate pipelines only: join and partition pipelines bake per-operator pointers into their programs)
  void share(const std::string& key) {
    if (!ctx || ctx->stream == nullptr) return;          // plan-time validation / precompilation: no device context
    auto it = ctx->shared_objects.find(key);
    if (it == ctx->shared_objects.end()) ctx->shared_objects.emplace(key, std::static_pointer_cast<void>(shared_state));
    else shared_state = std::static_pointer_cast<RunnerShared>(it->second);
  }
  DevScalars scal;
  int hot_wanted = 8;
  int64_t rows_seen = 0;                 // rows launched through this runner (specialisation threshold)
  uint64_t group_limit_cap = ~0ull;      // bounded aggregation: extra cap on the launch's group limit (see PipelineOp)
  // bounded aggregation: the limits the last guarded launch ran with (group table, pair sets), so the host can tell which
  // table a hand-back was for
  uint64_t last_group_limit = ~0ull, last_pair_limit[MAX_DISTINCT] = {};
  BufPtr distinct_params;                // device copy of the pair-set descriptors of both stages (PipelineAux::distinct)
  std::function<void(PipelineCompiler&, CompiledPipeline&)> custom_sink;   // build / partition sinks
  std::function<void(PipelineCompiler&, CompiledPipeline&)> pre_stages;    // probe ops injected before the stages

  void init(Ctx* c, const Schema& in) { ctx = c; in_schema = in; }   // no device work: specs can be validated without a GPU
  void ensure_scratch() { if (!scal.buf) scal.buf = dev_alloc_zero(ctx, 256); }

  std::shared_ptr<CompiledPipeline> compiled_for(const DevBatch& b, bool cold_variant = false) {
    std::vector<bool> sig;
    for (auto& c : b.cols) sig.push_back((bool)c.validity);
    std::vector<bool> cache_key = sig;
    cache_key.push_back(cold_variant);
    auto& cache = shared_state->cache;
    auto it = cache.find(cache_key);
    if (it != cache.end()) return it->second;
    auto cp = std::make_shared<CompiledPipeline>();
    cp->cold_variant = cold_variant;
    PipelineCompiler pc(in_schema, sig);
    if (pre_stages) pre_stages(pc, *cp);
    bool agg = false;
    for (auto& st : stages) {
      SG_CHECK(!agg, SAILGPU_ERR_INVALID, "aggregate must be the last stage of a pipeline");
      if (st.kind == StageSpec::Filter) {
        pc.add_filter(st.predicate);
        if (st.has_projection) pc.set_projection(st.projection);
      } else if (st.kind == StageSpec::Projection) {
        pc.set_exprs(st.exprs);
      } else {
        pc.finish_aggregate(*cp, st);
        agg = true;
      }
    }
    if (!agg) { if (custom_sink) custom_sink(pc, *cp); else pc.finish_store_or_compact(*cp); }
    int hot = 0;
    if (agg) hot = cp->agg.n_keys == 0 ? 1 : hot_wanted;
    pc.finalize(*cp, ctx, hot);
    cache[cache_key] = cp;
    if (getenv("SAILGPU_DUMP")) dump_pipeline(*cp);
    return cp;
  }

  DevProgram& program_for(const std::shared_ptr<CompiledPipeline>& cp) {
    auto& programs = shared_state->programs;
    auto it = programs.find(cp.get());
    if (it == programs.end()) {
      DevProgram dp;
      size_t lit_bytes = 0;
      for (auto& s : cp->literals) lit_bytes += (s.size() + 15) & ~(size_t)15;
      dp.literals = dev_alloc(ctx, lit_bytes + 16);
      std::vector<uint8_t> blob(lit_bytes + 16, 0);
      size_t off = 0;
      for (auto& s : cp->literals) {
        memcpy(blob.data() + off, s.data(), s.size());
        dp.literal_ptrs.push_back(reinterpret_cast<uint64_t>(dp.literals->ptr) + off);
        off += (s.size() + 15) & ~(size_t)15;
      }
      if (!cp->literals.empty()) {
        SG_CUDA(cudaMemcpyAsync(dp.literals->ptr, blob.data(), blob.size(), cudaMemcpyHostToDevice, ctx->stream));
        stream_sync(ctx);   // host blob goes out of scope
      }
      for (auto& fx : cp->literal_fixups) cp->prog[(size_t)fx.first].imm1 = dp.literal_ptrs[(size_t)fx.second];
      it = programs.emplace(cp.get(), std::move(dp)).first;
    }
    return it->second;
  }

  // fills inputs + common fields; caller fills sink buffers; then launch()
  void prepare(PipelineParams& P, const CompiledPipeline& cp, const DevBatch& b, int64_t row0, int64_t nrows) {
    ensure_scratch();
    memset(&P, 0, sizeof(P));
    P.n_rows = nrows;
    P.tile_rows = cp.rpt * NT;
    P.n_inputs = (int)cp.inputs.size();
    P.n_inst = (int)cp.prog.size();
    P.sink = cp.sink;
    P.arena_bytes = cp.arena_bytes;
    P.mask_slot = cp.mask_slot;
    P.error_flag = scal.error();
    P.n_probes = cp.n_probes;
    bool tma = true;
    SG_CHECK(row0 % 1024 == 0, SAILGPU_ERR_INVALID, "chunk offset must be a multiple of 1024 rows");
    for (size_t i = 0; i < cp.inputs.size(); ++i) {
      const InputReg& r = cp.inputs[i];
      const DevColumn& c = b.cols[(size_t)r.col];
      const uint8_t* base = static_cast<const uint8_t*>(r.validity ? c.validity->ptr : c.data->ptr);
      base += r.width ? row0 * r.width : row0 / 8;
      P.in[i].data = base;
      P.in[i].slot = (uint32_t)r.slot;
      P.in[i].width = r.width;
      P.in[i].tma_ok = (reinterpret_cast<uint64_t>(base) & 15) == 0 ? 1 : 0;
      tma &= P.in[i].tma_ok != 0;
    }
    P.use_tma = tma ? 1 : 0;
  }

  static uint32_t rs(uint32_t off, uint32_t add) { return off == NO_SLOT ? NO_SLOT : (off & 0x7FFFFFFFu) + ((off >> 31) ? add : 0u); }
  static void rs_key(KeyDesc& k, uint32_t add) { k.slot = rs(k.slot, add); k.valid_slot = rs(k.valid_slot, add); }

  // Builds the kernel argument block: program, descriptors and parameters resolved for both stages.
  void launch(PipelineParams& P, const std::shared_ptr<CompiledPipeline>& cp, const PipelineAux* aux_host, Metrics& m) {
    program_for(cp);
    const int64_t n_tiles = P.tile_list ? P.n_list : (P.n_rows + P.tile_rows - 1) / P.tile_rows;
    if (n_tiles == 0) return;
    P.prog = nullptr;
    auto K = std::make_unique<KernelArgs>();
    memset(K.get(), 0, sizeof(KernelArgs));
    const int n_distinct = aux_host ? aux_host->n_distinct : 0;
    std::vector<AggParams> dist(n_distinct ? (size_t)(2 * MAX_DISTINCT) : 0);
    for (int st = 0; st < 2; ++st) {
      const uint32_t add = (uint32_t)st * cp->stage_bytes;
      PipelineParams& Q = K->P[st];
      Q = P;
      Q.mask_slot = rs(P.mask_slot, add);
      for (int i = 0; i < Q.n_inputs; ++i) Q.in[i].slot = rs(P.in[i].slot, add);
      for (int j = 0; j < Q.n_out; ++j) { Q.out[j].slot = rs(P.out[j].slot, add); Q.out[j].valid_slot = rs(P.out[j].valid_slot, add); }
      for (size_t i = 0; i < cp->prog.size(); ++i) {
        VmInst I = cp->prog[i];
        I.dst = rs(I.dst, add); I.a = rs(I.a, add); I.b = rs(I.b, add); I.c = rs(I.c, add);
        K->prog[st][i] = I;
      }
      if (aux_host) {
        PipelineAux& A = K->aux[st];
        A = *aux_host;
        for (int i = 0; i < A.agg.n_keys; ++i) rs_key(A.agg.keys[i], add);
        for (int w = 0; w < A.agg.key_words; ++w) { A.agg.kwords[w].slot = rs(A.agg.kwords[w].slot, add); A.agg.kwords[w].valid_slot = rs(A.agg.kwords[w].valid_slot, add); }
        for (int j = 0; j < A.agg.n_accs; ++j) {
          AccDesc& d = A.agg.accs[j];
          d.value_slot = rs(d.value_slot, add); d.valid_slot = rs(d.valid_slot, add); d.n_slot = rs(d.n_slot, add); d.mean_slot = rs(d.mean_slot, add);
        }
        for (int j = 0; j < A.agg.n_accs && j < REG_ACCS; ++j) if (A.agg.rload[j].mode) A.agg.rload[j].slot = rs(A.agg.rload[j].slot, add);
        for (int i = 0; i < A.build.n_keys; ++i) rs_key(A.build.keys[i], add);
        for (int i = 0; i < A.part.n_keys; ++i) rs_key(A.part.keys[i], add);
        A.part.pid_slot = rs(A.part.pid_slot, add);
        for (int q = 0; q < MAX_PROBES; ++q) {
          for (int i = 0; i < A.probe[q].n_keys; ++i) rs_key(A.probe[q].keys[i], add);
          A.probe[q].rowid_slot = rs(A.probe[q].rowid_slot, add);
          A.probe[q].match_slot = rs(A.probe[q].match_slot, add);
        }
        for (int d = 0; d < n_distinct; ++d) {      // aux_host->distinct: the host copy of the descriptors
          AggParams& D = dist[(size_t)(st * MAX_DISTINCT + d)];
          D = aux_host->distinct[d];
          for (int i = 0; i < D.n_keys; ++i) rs_key(D.keys[i], add);
        }
      }
    }
    // Specialised kernel (jit.cu) once the operator has seen enough rows to pay for its compilation, or at once when the
    // kernel is already cached; everything else -- and every pipeline the specialiser does not cover -- is interpreted.
    rows_seen += P.n_rows;
    std::shared_ptr<JitKernel> jk;
    if (jit_enabled() && P.use_tma && !cp->jit_failed) {
      jk = cp->jit_kernel;
      if (!jk) {
        try {
          if (!cp->jit_checked) {      // once per compiled pipeline: is it covered, and is its kernel already cached?
            cp->jit_checked = true;
            std::string why;
            if (!jit_supported(*cp, &why)) { cp->jit_failed = true; if (getenv("SAILGPU_JIT_VERBOSE")) fprintf(stderr, "[sailgpu jit] interpreted: %s\n", why.c_str()); }
            else if (jit_cached(*cp, ctx->max_smem)) jk = cp->jit_kernel = jit_get_kernel(*cp, ctx->max_smem);
          }
          if (!jk && !cp->jit_failed && rows_seen >= jit_min_rows()) jk = cp->jit_kernel = jit_get_kernel(*cp, ctx->max_smem);
        } catch (const Error& e) {
          cp->jit_failed = true;
          if (getenv("SAILGPU_JIT_VERBOSE") || getenv("SAILGPU_JIT_STRICT")) fprintf(stderr, "[sailgpu jit] not specialised: %s\n", e.what());
          if (getenv("SAILGPU_JIT_STRICT")) throw;
        }
      }
    }
    // resident CTAs per SM: what shared memory allows, then the matching register-budget variant of the kernel
    const int by_smem = std::max(1, (int)(ctx->max_smem / (cp->smem_bytes + 1024)));
    const char* fm = getenv("SAILGPU_MINB");
    const int minb = fm && *fm ? atoi(fm) : std::min(by_smem, cp->sink == SINK_AGG ? (cp->cold_variant ? 4 : 2) : (cp->sink == SINK_BUILD || cp->n_probes > 0) ? 4 : 3);
    const int per_sm = jk ? jk->ctas_per_sm : std::max(1, std::min(by_smem, pipeline_max_ctas_per_sm(cp->rpt, minb, cp->smem_bytes, cp->sink, cp->cold_variant)));
    const int grid = (int)std::min<int64_t>(n_tiles, (int64_t)ctx->sm_count * per_sm);
    if (cp->sink == SINK_AGG && aux_host && aux_host->agg.deferred) {
      // group limit of a bounded table: half the capacity minus what can still arrive from tiles in flight (a CTA acts
      // on a table-full reading that is up to two tiles old, so three tiles per CTA; a specialised kernel has its whole
      // stage ring in flight) and from the dictionary flushes
      const uint64_t cap = aux_host->agg.capacity_mask + 1;
      const uint64_t in_flight = jk ? (uint64_t)jk->stages + 1 : 3ull;
      const uint64_t slack = std::min<uint64_t>(in_flight * (uint64_t)grid * (uint64_t)P.tile_rows, (uint64_t)P.n_rows) + (uint64_t)grid * (uint64_t)std::max(0, cp->agg.hot_groups);
      const uint64_t limit = std::min<uint64_t>(cap / 2 > slack ? cap / 2 - slack : 0, group_limit_cap);
      for (int st = 0; st < 2; ++st)
        if (K->aux[st].agg.group_limit == ~0ull && cp->agg.n_keys > 0) K->aux[st].agg.group_limit = limit;     // one group never grows
      // a pair set gains at most one pair per row: only the rows in flight count
      const uint64_t pair_slack = std::min<uint64_t>(in_flight * (uint64_t)grid * (uint64_t)P.tile_rows, (uint64_t)P.n_rows);
      for (int d = 0; d < n_distinct; ++d) {
        const uint64_t dcap = dist[(size_t)d].capacity_mask + 1;
        last_pair_limit[d] = dcap / 2 > pair_slack ? dcap / 2 - pair_slack : 0;
        for (int st = 0; st < 2; ++st) dist[(size_t)(st * MAX_DISTINCT + d)].group_limit = last_pair_limit[d];
      }
      last_group_limit = K->aux[0].agg.group_limit;
    }
    if (n_distinct) {
      if (!distinct_params) distinct_params = dev_alloc(ctx, dist.size() * sizeof(AggParams));
      SG_CUDA(cudaMemcpyAsync(distinct_params->ptr, dist.data(), dist.size() * sizeof(AggParams), cudaMemcpyHostToDevice, ctx->stream));
      for (int st = 0; st < 2; ++st) K->aux[st].distinct = static_cast<const AggParams*>(distinct_params->ptr) + st * MAX_DISTINCT;
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    const bool timed = timing_enabled();
    if (timed) { SG_CUDA(cudaEventCreate(&e0)); SG_CUDA(cudaEventCreate(&e1)); SG_CUDA(cudaEventRecord(e0, ctx->stream)); }
    if (jk) { jit_launch(*jk, *K, grid, ctx->stream); m.jit_launches++; }
    else SG_CUDA(launch_pipeline(*K, cp->rpt, cp->n_stages, cp->smem_bytes, grid, minb, ctx->stream));
    if (timed) { SG_CUDA(cudaEventRecord(e1, ctx->stream)); m.pending.emplace_back(e0, e1); }
    m.kernel_launches++;
    m.pipeline_launches++;
  }
};


// Runs a STORE / COMPACT pipeline over one batch and returns the output batch.
// `tile_offsets` (with `known_out_rows`): COMPACT without look-back, every tile's output position precomputed (two-pass filter).
inline BatchPtr run_streaming(PipelineRunner& run, Ctx* ctx, const BatchPtr& b, Metrics& m, const PipelineAux* aux_host, const std::vector<BufPtr>& extra_heaps,
                              const unsigned long long* tile_offsets = nullptr, int64_t known_out_rows = -1) {
  auto cp = run.compiled_for(*b);
  auto out = std::make_shared<DevBatch>();
  const int64_t n = b->rows;
  PipelineParams P;
  run.prepare(P, *cp, *b, 0, n);
  const bool compact = cp->sink == SINK_COMPACT;
  P.n_out = (int)cp->outs.size();
  SG_CHECK(P.n_out <= MAX_OUTPUTS, SAILGPU_ERR_UNSUPPORTED, "more than " + std::to_string(MAX_OUTPUTS) + " output columns");
  std::vector<BufPtr> valid_tmp((size_t)P.n_out), bool_tmp((size_t)P.n_out);
  std::vector<BufPtr> all_heaps;
  for (auto& c : b->cols) if (c.type.is_string()) for (auto& h : c.heaps) all_heaps.push_back(h);
  for (auto& h : extra_heaps) all_heaps.push_back(h);
  for (int j = 0; j < P.n_out; ++j) {
    OutputCol o = cp->outs[(size_t)j];
    DevColumn c; c.type = cp->out_types[(size_t)j]; c.arrow_is_utf8 = c.type.id == TypeId::Utf8;
    if (o.width) { c.data = dev_alloc(ctx, (size_t)n * o.width); o.data = static_cast<uint8_t*>(c.data->ptr); }
    else if (compact) { bool_tmp[(size_t)j] = dev_alloc(ctx, (size_t)n); o.data = static_cast<uint8_t*>(bool_tmp[(size_t)j]->ptr); }
    else { c.data = dev_alloc_zero(ctx, (size_t)((n + 31) / 32 * 4)); o.data = static_cast<uint8_t*>(c.data->ptr); }
    if (o.valid_slot != NO_SLOT) {
      if (compact) { valid_tmp[(size_t)j] = dev_alloc(ctx, (size_t)n); o.valid_bytes = static_cast<uint8_t*>(valid_tmp[(size_t)j]->ptr); }
      else { c.validity = dev_alloc_zero(ctx, (size_t)((n + 31) / 32 * 4)); o.valid_bytes = static_cast<uint8_t*>(c.validity->ptr); c.null_count = -1; }
    }
    if (c.type.is_string()) c.heaps = all_heaps;
    P.out[j] = o;
    out->cols.push_back(c);
  }
  BufPtr status;
  if (compact && tile_offsets) {
    P.tile_offsets = tile_offsets;
  } else if (compact) {
    const int64_t n_tiles = (n + P.tile_rows - 1) / P.tile_rows;
    status = dev_alloc_zero(ctx, (size_t)(n_tiles + 1) * 8);
    P.tile_status = static_cast<unsigned long long*>(status->ptr);
    P.ticket = run.scal.ticket();
    P.out_count = run.scal.out_count();
    SG_CUDA(cudaMemsetAsync(static_cast<uint8_t*>(run.scal.buf->ptr) + 8, 0, 16, ctx->stream));
  }
  run.launch(P, cp, aux_host, m);
  int64_t out_rows = n;
  if (compact) {
    unsigned long long cnt = (unsigned long long)known_out_rows;
    if (!tile_offsets) SG_CUDA(cudaMemcpyAsync(&cnt, run.scal.out_count(), 8, cudaMemcpyDeviceToHost, ctx->stream));
    check_device_error(ctx, run.scal.error());   // synchronises
    out_rows = (int64_t)cnt;
    for (int j = 0; j < P.n_out; ++j) {
      DevColumn& c = out->cols[(size_t)j];
      if (bool_tmp[(size_t)j]) {
        c.data = dev_alloc_zero(ctx, (size_t)((out_rows + 31) / 32 * 4));
        SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(bool_tmp[(size_t)j]->ptr), static_cast<uint32_t*>(c.data->ptr), out_rows, nullptr, ctx->stream));
      }
      if (valid_tmp[(size_t)j]) {
        c.validity = dev_alloc_zero(ctx, (size_t)((out_rows + 31) / 32 * 4));
        SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(valid_tmp[(size_t)j]->ptr), static_cast<uint32_t*>(c.validity->ptr), out_rows, nullptr, ctx->stream));
        c.null_count = -1;
      }
    }
    if (!bool_tmp.empty() || !valid_tmp.empty()) stream_sync(ctx);
  } else {
    check_device_error(ctx, run.scal.error());
  }
  out->rows = out_rows;
  for (auto& c : out->cols) c.length = out_rows;
  return out;
}


}  // namespace sg
