// engine.cu -- PipelineOp: FilterExec / ProjectionExec / AggregateExec (and fused chains of them)
// executed by the tile-pipeline kernel.  Mirrors DataFusion's operator contract as Sail uses it
// (SURVEY.md section 8b): streaming operators emit one output batch per input batch; the aggregate
// consumes its whole input and emits at end of stream; NULL predicate rows are dropped; schemas are
// fixed at construction.
#include "runner.hpp"

namespace sg {

// Copies the first `words` words of an operator's scalars into mapped host memory and zeroes the hand-back counter of the next
// launch: one tiny launch between two aggregate launches instead of a device->host copy and a memset.
__global__ void agg_counters_kernel(const unsigned long long* __restrict__ scal, unsigned long long* host, int words, unsigned long long* zero) {
  if (threadIdx.x < words) host[threadIdx.x] = scal[threadIdx.x];
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0 && zero) *zero = 0;
}


// ------------------------------------------------------------------------------------------------
// spec parsing
// ------------------------------------------------------------------------------------------------
// An aggregate's "distinct": true (DataFusion's AggregateFunctionExpr::is_distinct).  count / sum / avg over one argument of a
// single-mode aggregate run as accumulators behind a per-pair gate (compiler.cu finish_aggregate); for min / max the flag
// changes nothing and is dropped, as in DataFusion.  Everything else is refused here, while planning.
static int pair_key_words(const DataType& t) { return t.is_string() || (t.is_decimal() && t.precision > 18) ? 2 : 1; }
static void check_distinct(const StageSpec& st, StageSpec::Agg& ag, const Json* args, std::set<std::string>* distinct_args) {
  const std::string what = ag.fn + "(DISTINCT) '" + ag.name + "'";
  SG_CHECK(st.mode == "single", SAILGPU_ERR_UNSUPPORTED, what + " in mode '" + st.mode + "' is not supported on the GPU path: DataFusion's partial state of a DISTINCT aggregate is a List column");
  const size_t n_args = args && args->kind == Json::Arr ? args->a.size() : 0;
  SG_CHECK(n_args > 0, SAILGPU_ERR_INVALID, what + " needs an argument");
  SG_CHECK(n_args == 1, SAILGPU_ERR_UNSUPPORTED, what + " over more than one argument is not supported on the GPU path");
  if (ag.fn == "min" || ag.fn == "max") return;
  SG_CHECK(ag.fn == "count" || ag.fn == "sum" || ag.fn == "avg", SAILGPU_ERR_UNSUPPORTED, "aggregate function '" + ag.fn + "' with DISTINCT");
  const DataType& t = ag.arg->type;
  SG_CHECK(!t.is_float() && t.id != TypeId::Bool, SAILGPU_ERR_UNSUPPORTED, what + " over " + t.str() + " is not supported on the GPU path");
  // the pair set's key: a null-mask word, the group keys, the argument (compiler.cu gate_for)
  int words = 1 + pair_key_words(t);
  for (auto& g : st.group_exprs) words += pair_key_words(g->type);
  SG_CHECK((int)st.group_exprs.size() + 1 <= MAX_KEYS && words <= MAX_KEY_WORDS, SAILGPU_ERR_UNSUPPORTED,
           what + ": the grouping columns and the argument take more than " + std::to_string(MAX_KEYS) + " columns or " + std::to_string(MAX_KEY_WORDS * 8) + " bytes of pair key");
  distinct_args->insert(ag.arg->key());
  SG_CHECK((int)distinct_args->size() <= MAX_DISTINCT, SAILGPU_ERR_UNSUPPORTED, "more than " + std::to_string(MAX_DISTINCT) + " DISTINCT arguments in one aggregate");
  ag.distinct = true;
}

StageSpec parse_stage(const Json& j, const Schema& in, Schema* out) {
  StageSpec st;
  const std::string op = j.at("op").as_str();
  if (op == "filter") {
    st.kind = StageSpec::Filter;
    st.predicate = parse_expr(j.at("predicate"), in);
    SG_CHECK(st.predicate->type.id == TypeId::Bool, SAILGPU_ERR_INVALID, "filter predicate must be boolean");
    const Json* p = j.find("projection");
    if (p && !p->is_null()) {
      st.has_projection = true;
      for (auto& x : p->a) {
        int i = (int)x.as_int();
        SG_CHECK(i >= 0 && i < (int)in.size(), SAILGPU_ERR_INVALID, "filter projection index out of range");
        st.projection.push_back(i);
        out->push_back(in[(size_t)i]);
      }
    } else *out = in;
  } else if (op == "projection") {
    st.kind = StageSpec::Projection;
    for (auto& x : j.at("exprs").a) {
      ExprPtr e = parse_expr(x.at("expr"), in);
      st.exprs.push_back(e);
      st.names.push_back(x.at("name").as_str());
      out->push_back({st.names.back(), e->type, e->nullable});
    }
  } else if (op == "aggregate") {
    st.kind = StageSpec::Aggregate;
    const Json* md = j.find("mode");
    st.mode = md ? md->as_str() : "single";
    SG_CHECK(st.mode == "single" || st.mode == "partial" || st.mode == "final" || st.mode == "final_partitioned", SAILGPU_ERR_INVALID,
             "aggregate mode '" + st.mode + "'");
    const bool merging = st.mode == "final" || st.mode == "final_partitioned";
    for (auto& g : j.at("group_by").a) {
      ExprPtr e = parse_expr(g.at("expr"), in);
      st.group_exprs.push_back(e);
      st.group_names.push_back(g.at("name").as_str());
      out->push_back({st.group_names.back(), e->type, e->nullable});
    }
    size_t state_col = st.group_exprs.size();
    std::set<std::string> distinct_args;
    for (auto& a : j.at("aggs").a) {
      StageSpec::Agg ag;
      ag.fn = a.at("fn").as_str();
      ag.name = a.at("name").as_str();
      const Json* it = a.find("input_type");
      if (it && !it->is_null()) ag.input_type = parse_type(it->as_str());
      const Json* args = a.find("args");
      if (!merging && args && args->kind == Json::Arr && !args->a.empty()) { ag.arg = parse_expr(args->a[0], in); ag.has_arg = true; ag.input_type = ag.arg->type; }
      SG_CHECK(ag.fn == "count" || ag.has_arg || merging, SAILGPU_ERR_INVALID, "aggregate '" + ag.fn + "' needs an argument");
      const Json* ds = a.find("distinct");
      if (ds && !ds->is_null()) {
        SG_CHECK(ds->kind == Json::Bool, SAILGPU_ERR_INVALID, "aggregate '" + ag.name + "': \"distinct\" must be true or false");
        if (ds->b) check_distinct(st, ag, args, &distinct_args);
      }
      SG_CHECK(ag.fn == "count" || ag.input_type.id != TypeId::Null, SAILGPU_ERR_INVALID, "aggregate '" + ag.name + "' needs input_type in final mode");
      AggTypes at = agg_types(ag.fn, ag.fn == "count" ? T(TypeId::Int64) : ag.input_type);
      if (merging) {
        for (size_t k = 0; k < at.state.size(); ++k) {
          SG_CHECK(state_col + k < in.size(), SAILGPU_ERR_INVALID, "final aggregate: input has too few state columns");
          const DataType& have = in[state_col + k].type;
          SG_CHECK(have == at.state[k] || (have.id == TypeId::Int64 && at.state[k].id == TypeId::UInt64) || (have.id == TypeId::UInt64 && at.state[k].id == TypeId::Int64),
                   SAILGPU_ERR_INVALID, "final aggregate: state column " + std::to_string(state_col + k) + " is " + have.str() + ", expected " + at.state[k].str());
        }
      }
      state_col += at.state.size();
      if (st.mode == "partial") {
        if (ag.fn == "avg") { out->push_back({ag.name + "[count]", at.state[0], false}); out->push_back({ag.name + "[sum]", at.state[1], true}); }
        else if (is_variance_fn(ag.fn)) {
          out->push_back({ag.name + "[count]", at.state[0], false});
          out->push_back({ag.name + "[mean]", at.state[1], false});
          out->push_back({ag.name + "[m2]", at.state[2], false});
        }
        else out->push_back({ag.name + "[" + ag.fn + "]", at.state[0], ag.fn != "count"});
      } else {
        out->push_back({ag.name, at.final_type, ag.fn != "count"});
      }
      st.aggs.push_back(ag);
    }
  } else {
    fail(SAILGPU_ERR_UNSUPPORTED, "operator '" + op + "' cannot be part of a fused pipeline");
  }
  return st;
}

// throws the error a kernel raised in `f` (the value of the device flag at `dev_flag`), after clearing the flag
void raise_device_error(Ctx* ctx, uint32_t* dev_flag, uint32_t f) {
  if (!f) return;
  SG_CUDA(cudaMemsetAsync(dev_flag, 0, 4, ctx->stream));
  if (f & ERR_DIV_ZERO) fail(SAILGPU_ERR_ARITHMETIC, "Divide by zero");
  if (f & ERR_OVERFLOW) fail(SAILGPU_ERR_ARITHMETIC, "Arithmetic overflow");
  if (f & ERR_TABLE_FULL) fail(SAILGPU_ERR_CUDA, "hash table overflow");
  fail(SAILGPU_ERR_UNSUPPORTED, "unsupported value encountered on device");
}

void check_device_error(Ctx* ctx, uint32_t* dev_flag) {
  uint32_t f = 0;
  SG_CUDA(cudaMemcpyAsync(&f, dev_flag, 4, cudaMemcpyDeviceToHost, ctx->stream));
  stream_sync(ctx);
  raise_device_error(ctx, dev_flag, f);
}

// ------------------------------------------------------------------------------------------------
// PipelineOp
// ------------------------------------------------------------------------------------------------
struct AggTable {
  BufPtr table, state, occ;
  uint64_t capacity = 0;
};

struct PipelineOp : Op {
  PipelineRunner run;
  bool has_agg = false;
  StageSpec* agg_stage = nullptr;
  AggTable tab;
  std::shared_ptr<CompiledPipeline> agg_cp;   // all launches of an aggregate must share one layout
  std::deque<BatchPtr> ready;
  std::vector<BufPtr> kept_heaps;
  bool input_done = false, emitted = false;

  void collect_heaps(const DevBatch& b) {
    for (auto& c : b.cols)
      if (c.type.is_string()) for (auto& h : c.heaps) kept_heaps.push_back(h);
  }

  void push(int input, const BatchPtr& b) override {
    SG_CHECK(input == 0, SAILGPU_ERR_INVALID, "operator has one input");
    SG_CHECK(!input_done, SAILGPU_ERR_STATE, "push after finish_input");
    const uint64_t t0 = now_ns();
    m.input_rows += (uint64_t)b->rows; m.input_batches++;
    if (has_agg) { collect_heaps(*b); push_agg(b); }
    else if (const std::vector<int>* cols = rename_only()) {
      // a ProjectionExec of plain column references (the `expr=[_0@0 as #9, _3@1 as #12]` nodes over every scan in the reference's
      // plans) moves no data: the output batch shares the input's buffers, as DataFusion's Arc-cloned arrays do
      auto out = std::make_shared<DevBatch>();
      out->rows = b->rows;
      for (int c : *cols) out->cols.push_back(b->cols[(size_t)c]);
      ready.push_back(out);
    }
    else ready.push_back(run_stream(b));
    m.elapsed_compute_ns += now_ns() - t0;
  }
  // the input column of every output when the whole pipeline is projections of bare column references, else null
  int rename_state = -1;      // -1: not analysed yet, 0: no, 1: yes
  std::vector<int> rename_cols;
  const std::vector<int>* rename_only() {
    if (rename_state < 0) {
      rename_state = 0;
      std::vector<int> cur;
      bool ok = !run.stages.empty();
      for (size_t si = 0; ok && si < run.stages.size(); ++si) {
        const StageSpec& st = run.stages[si];
        if (st.kind != StageSpec::Projection) { ok = false; break; }
        std::vector<int> next;
        for (auto& e : st.exprs) {
          if (e->kind != Expr::Col) { ok = false; break; }
          next.push_back(si == 0 ? e->col : cur[(size_t)e->col]);
        }
        cur.swap(next);
      }
      if (ok) { rename_cols = cur; rename_state = 1; }
    }
    return rename_state == 1 ? &rename_cols : nullptr;
  }
  void finish(int input) override {
    SG_CHECK(input == 0, SAILGPU_ERR_INVALID, "operator has one input");
    input_done = true;
  }
  bool pull(BatchPtr* out) override {
    *out = nullptr;
    if (has_agg) {
      // the aggregate's result once the input ended; before that only what partitioned mode emitted early (partial mode)
      if (input_done && !emitted) {
        const uint64_t t0 = now_ns();
        if (tab.capacity) current_groups();      // resolves the launches in flight first: they may still spill
        if (spilled.empty()) ready.push_back(extract_agg());
        else finish_partitioned();
        m.elapsed_compute_ns += now_ns() - t0;
        emitted = true;
      }
      if (!ready.empty()) {
        *out = ready.front(); ready.pop_front();
        m.output_rows += (uint64_t)(*out)->rows; m.output_batches++;
      }
      return !(emitted && ready.empty());
    }
    if (!ready.empty()) {
      *out = ready.front(); ready.pop_front();
      m.output_rows += (uint64_t)(*out)->rows; m.output_batches++;
      return !(input_done && ready.empty());
    }
    return !input_done;
  }

  // ---- two-pass filter ---------------------------------------------------------------------------
  // An order-preserving single-pass compaction chains every tile to all earlier ones (decoupled look-back), and since a
  // tile only knows its count after evaluating the predicate the chain runs at the pace of the slowest resident tile
  // (the largest share of the FilterExec kernel's stall samples).  Large batches therefore take two passes: pass 1
  // reads only the predicate's columns and stores the mask (1 bit / row); the per-tile popcounts are scanned; pass 2
  // reads the projected columns + mask and stores every tile at its known offset, tiles in any order.
  static constexpr int64_t TWO_PASS_MIN_ROWS = 1 << 18;
  PipelineRunner mask_run, sel_run;
  bool two_pass_ready = false;
  std::string share_key;
  void setup_two_pass() {
    const Schema& in = run.in_schema;
    mask_run.init(ctx, in);
    if (!share_key.empty()) mask_run.share(share_key + "#mask");
    StageSpec f; f.kind = StageSpec::Filter; f.predicate = run.stages[0].predicate;
    mask_run.stages.push_back(f);
    mask_run.custom_sink = [](PipelineCompiler& pc, CompiledPipeline& cp) { pc.finish_mask_store(cp); };
    Schema in2 = in;
    Field mf; mf.name = "__mask"; mf.type.id = TypeId::Bool; mf.nullable = false;
    in2.push_back(mf);
    sel_run.init(ctx, in2);
    if (!share_key.empty()) sel_run.share(share_key + "#select");
    sel_run.stages = run.stages;
    StageSpec& s0 = sel_run.stages[0];
    auto me = std::make_shared<Expr>(); me->kind = Expr::Col; me->col = (int)in.size(); me->type.id = TypeId::Bool; me->nullable = false;
    s0.predicate = me;
    if (!s0.has_projection) { s0.has_projection = true; s0.projection.clear(); for (size_t i = 0; i < in.size(); ++i) s0.projection.push_back((int)i); }
    two_pass_ready = true;
  }
  bool two_pass_applies(const BatchPtr& b) const {
    const char* mn = getenv("SAILGPU_TWO_PASS_MIN");     // rows from which a filter runs in two passes (tests lower it; "off" disables)
    if (mn && !strcmp(mn, "off")) return false;
    const int64_t min_rows = mn && *mn ? atoll(mn) : TWO_PASS_MIN_ROWS;
    return !has_agg && !run.stages.empty() && run.stages[0].kind == StageSpec::Filter && b->rows >= min_rows;
  }
  BatchPtr run_two_pass(const BatchPtr& b) {
    if (!two_pass_ready) setup_two_pass();
    BatchPtr mb = run_streaming(mask_run, ctx, b, m, nullptr, {});
    auto b2 = std::make_shared<DevBatch>(*b);
    b2->cols.push_back(mb->cols[0]);
    auto cp2 = sel_run.compiled_for(*b2);
    const int tile_rows = cp2->rpt * NT;
    const int64_t n = b->rows, n_tiles = (n + tile_rows - 1) / tile_rows;
    BufPtr counts = dev_alloc_zero(ctx, (size_t)(n_tiles + 1) * 4), offs = dev_alloc(ctx, (size_t)(n_tiles + 1) * 8), scratch = dev_alloc(ctx, 1026 * 8);
    SG_CUDA(launch_tile_popcount(static_cast<const uint32_t*>(mb->cols[0].data->ptr), n, tile_rows, n_tiles, static_cast<uint32_t*>(counts->ptr), ctx->stream));
    SG_CUDA(launch_exclusive_scan_u32(static_cast<const uint32_t*>(counts->ptr), n_tiles + 1, static_cast<uint64_t*>(offs->ptr), static_cast<uint64_t*>(scratch->ptr), ctx->stream));
    unsigned long long total = 0;
    SG_CUDA(cudaMemcpyAsync(&total, static_cast<const uint64_t*>(offs->ptr) + n_tiles, 8, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    m.kernel_launches += 4;
    return run_streaming(sel_run, ctx, b2, m, nullptr, {}, static_cast<const unsigned long long*>(offs->ptr), (int64_t)total);
  }

  BatchPtr run_stream(const BatchPtr& b) {
    if (two_pass_applies(b)) return run_two_pass(b);
    return run_streaming(run, ctx, b, m, nullptr, {});
  }

  // ---- aggregate ------------------------------------------------------------------------------
  // The group table is sized for the groups the operator expects, not for its input rows.  Every launch carries a group
  // limit (half the capacity minus what tiles in flight could still add); CTAs that see the table above it stop taking
  // tiles and append the ones they still owned to a deferred list.  If tiles were handed back the host grows the table by
  // the observed groups-per-row ratio, rehashes, and re-launches over the list -- with the pipeline variant compiled for
  // the global table alone when the input turned out to have many groups.
  //
  // Launches are pipelined one deep: after queueing the launch of batch k, the host queues an asynchronous copy of the
  // counters (error flag, groups, both hand-back counts) into pinned memory and only then waits for the copy made after
  // batch k-1.  The device already has batch k to work on, so that wait costs it nothing.  When k-1 handed nothing back
  // and raised nothing, that is all.  Otherwise the host drains the stream and resolves k-1 and k together: a rehash
  // or layout migration must never run on a group count older than the last launch.  Each of the two launches in
  // flight has its own hand-back counter and list; the operator holds at most those two input batches.
  static constexpr uint64_t MIN_CAPACITY = 1ull << 22, MAX_CAPACITY = 1ull << 28;
  static constexpr uint64_t CARD_MANY_GROUPS = 256, HOT_GROUP_LIMIT = 1 << 16;
  static uint64_t min_capacity() { const char* v = getenv("SAILGPU_AGG_MIN_CAPACITY"); return v && *v ? next_pow2((uint64_t)atoll(v)) : MIN_CAPACITY; }
  // the most slots one table may have (tests lower it, so that partitioned mode is reached with few groups); the table of a
  // partition of partitioned mode (below) is sized to stay under MAX_CAPACITY whatever the ceiling was
  bool partition_of_parent = false;
  uint64_t max_capacity() const {
    const char* v = getenv("SAILGPU_AGG_MAX_CAPACITY");
    return v && *v && !partition_of_parent ? std::min(MAX_CAPACITY, next_pow2((uint64_t)atoll(v))) : MAX_CAPACITY;
  }
  bool use_cold = false;
  int64_t rows_in_table = 0;
  int64_t known_groups = -1;      // group count read (and error flag checked) once nothing was in flight any more, -1 = stale
  // a grouped launch whose hand-back has not been looked at yet; `slot` picks its hand-back counter and its counter copy
  struct InFlight { BatchPtr batch; std::shared_ptr<CompiledPipeline> cp; BufPtr deferred; int slot = 0; };
  std::deque<InFlight> inflight;
  int next_slot = 0;
  // what a counter copy holds: the first 56 bytes of the scalars (DevScalars: error @0, n_groups @24, hand-back counts @40, @48)
  struct Counters { uint32_t error; uint32_t pad_[5]; unsigned long long n_groups, cursor, n_def[2]; };
  static_assert(sizeof(Counters) == 56, "counter copy layout");
  Counters* counters = nullptr;        // two copies, in a pinned slot of the context (or on the heap when pinning failed)
  Counters* counters_dev = nullptr;    // the pinned slot as the device addresses it
  bool counters_pinned = false, next_zeroed = false;
  cudaEvent_t copied[2] = {nullptr, nullptr};

  ~PipelineOp() override {
    if (g_exiting.load()) return;
    for (cudaEvent_t e : copied) if (e) cudaEventDestroy(e);
    if (counters_pinned) pinned_slot_release(ctx, counters); else delete[] counters;
  }

  unsigned long long* n_deferred_ptr(int slot) { return reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(run.scal.buf->ptr) + 40 + 8 * slot); }

  // queues the copy of the counters into copy `slot` and marks its completion; `zero_next`: also zero the hand-back counter of
  // the other slot, which the next launch uses (launch_agg then skips its memset)
  void copy_counters(int slot, bool zero_next) {
    if (!counters) {
      static_assert(2 * sizeof(Counters) <= Ctx::PINNED_SLOT, "pinned slot too small");
      counters = static_cast<Counters*>(pinned_slot_acquire(ctx));
      counters_pinned = counters != nullptr;
      if (counters_pinned) SG_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&counters_dev), counters, 0));
      else counters = new Counters[2];
      for (auto& e : copied) SG_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    if (counters_pinned) {
      agg_counters_kernel<<<1, 32, 0, ctx->stream>>>(static_cast<const unsigned long long*>(run.scal.buf->ptr), reinterpret_cast<unsigned long long*>(&counters_dev[slot]),
                                                     (int)(sizeof(Counters) / 8), zero_next ? n_deferred_ptr(slot ^ 1) : nullptr);
      SG_CUDA(cudaGetLastError());
      m.kernel_launches++;
      next_zeroed = zero_next;
    } else {
      SG_CUDA(cudaMemcpyAsync(&counters[slot], run.scal.buf->ptr, sizeof(Counters), cudaMemcpyDeviceToHost, ctx->stream));
    }
    SG_CUDA(cudaEventRecord(copied[slot], ctx->stream));
  }

  void fill_table(AggParams& A) {
    A.table = static_cast<uint8_t*>(tab.table->ptr);
    A.state = static_cast<uint32_t*>(tab.state->ptr);
    A.occ = static_cast<uint32_t*>(tab.occ->ptr);
    A.capacity_mask = tab.capacity - 1;
    A.n_groups = run.scal.n_groups();
  }

  // (re)allocates the table with `cap` slots and moves the `groups` existing entries over
  void alloc_table(const AggParams& A0, uint64_t cap, uint64_t groups) {
    SG_CHECK(cap <= MAX_CAPACITY, SAILGPU_ERR_UNSUPPORTED, "aggregate needs more than 2^28 group slots");
    AggTable old = tab;
    tab.capacity = cap;
    tab.table = dev_alloc(ctx, (size_t)cap * A0.entry_words * 8);
    tab.state = dev_alloc_zero(ctx, (size_t)cap * 4);
    tab.occ = dev_alloc(ctx, (size_t)cap * 4);
    if (old.capacity && groups) {
      AggParams A = A0;
      fill_table(A);
      SG_CUDA(cudaMemsetAsync(run.scal.n_groups(), 0, 8, ctx->stream));
      SG_CUDA(launch_agg_rehash(A, static_cast<const uint8_t*>(old.table->ptr), static_cast<const uint32_t*>(old.occ->ptr), groups, run.scal.error(), ctx->stream));
      m.kernel_launches++;
    }
  }

  // ---- DISTINCT aggregates: pair sets ---------------------------------------------------------------
  // One set per DISTINCT argument (compiler.cu gate_for), a group table without accumulators.  A set is never emptied (not
  // by a spill either), grows like the group table -- bounded, with hand-backs -- and is not partitioned: past max_capacity()
  // the aggregate is refused.
  std::vector<AggTable> dsets;
  BufPtr dcounts;                      // the pair count of every set
  unsigned long long* pair_count(size_t d) { return static_cast<unsigned long long*>(dcounts->ptr) + d; }

  void alloc_set(size_t d, const AggParams& D0, uint64_t cap, uint64_t pairs) {
    SG_CHECK(cap <= max_capacity(), SAILGPU_ERR_UNSUPPORTED, "count(DISTINCT) needs more than " + std::to_string(max_capacity()) + " pair slots");
    AggTable old = dsets[d];
    AggTable& t = dsets[d];
    t.capacity = cap;
    t.table = dev_alloc(ctx, (size_t)cap * D0.entry_words * 8);
    t.state = dev_alloc_zero(ctx, (size_t)cap * 4);
    t.occ = dev_alloc(ctx, (size_t)cap * 4);
    if (old.capacity && pairs) {
      AggParams D = D0;
      fill_set(D, d);
      SG_CUDA(cudaMemsetAsync(pair_count(d), 0, 8, ctx->stream));
      SG_CUDA(launch_agg_rehash(D, static_cast<const uint8_t*>(old.table->ptr), static_cast<const uint32_t*>(old.occ->ptr), pairs, run.scal.error(), ctx->stream));
      m.kernel_launches++;
    }
  }
  void fill_set(AggParams& D, size_t d) {
    const AggTable& t = dsets[d];
    D.table = static_cast<uint8_t*>(t.table->ptr);
    D.state = static_cast<uint32_t*>(t.state->ptr);
    D.occ = static_cast<uint32_t*>(t.occ->ptr);
    D.capacity_mask = t.capacity - 1;
    D.n_groups = pair_count(d);
    D.group_limit = ~0ull;           // launch() derives it from the grid
  }

  // one launch over all tiles of `b` (list == null) or over the listed tiles; tiles handed back land in `deferred_out`
  void launch_agg(const std::shared_ptr<CompiledPipeline>& cp, const DevBatch& b, const BufPtr& list, int64_t n_list, const BufPtr& deferred_out, int slot) {
    PipelineParams P;
    run.prepare(P, *cp, b, 0, b.rows);
    if (list) { P.tile_list = static_cast<const uint32_t*>(list->ptr); P.n_list = n_list; }
    PipelineAux aux;
    memset(&aux, 0, sizeof(aux));
    aux.agg = cp->agg;
    fill_table(aux.agg);
    std::vector<AggParams> sets = cp->distinct;       // host copy: launch() rebases it per stage and uploads it
    for (size_t d = 0; d < sets.size(); ++d) fill_set(sets[d], d);
    aux.distinct = sets.data();
    aux.n_distinct = (int32_t)sets.size();
    if (deferred_out) {
      if (!(next_zeroed && !list)) SG_CUDA(cudaMemsetAsync(n_deferred_ptr(slot), 0, 8, ctx->stream));
      next_zeroed = false;
      aux.agg.deferred = static_cast<uint32_t*>(deferred_out->ptr);
      aux.agg.n_deferred = n_deferred_ptr(slot);
      const char* fl = getenv("SAILGPU_AGG_FIRST_LIMIT");      // tests: force an early hand-back on the first pass
      aux.agg.group_limit = (!list && fl && *fl) ? (unsigned long long)atoll(fl) : ~0ull;   // ~0: launch() derives it from the grid
      // the dictionary variant is only worth running while there are few groups: it hands back early, and the
      // re-launch (many-groups variant, table sized by the observed ratio) takes over
      run.group_limit_cap = (cp->cold_variant || list) ? ~0ull : HOT_GROUP_LIMIT;      // re-launches over a list always make progress
    }
    run.launch(P, cp, &aux, m);
  }

  // ---- validity signatures ------------------------------------------------------------------------
  // The entry layout (null-mask word, seen bits, one counter per nullable avg/count argument) follows from which input
  // columns carry validity buffers, and Arrow batches of one stream differ in that (a producer drops the bitmap of a
  // batch without nulls).  The operator therefore keeps the union of the signatures it has seen: a batch that lacks a
  // bitmap of the union gets an all-ones one, and when a batch widens the union the table is carried over to the wider
  // layout (migrate_layout).  DataFusion's accumulators take `null_count == 0` fast paths per batch the same way.
  std::vector<bool> sticky_sig;
  BufPtr ones; size_t ones_bytes = 0;

  BatchPtr with_union_signature(const BatchPtr& b, bool* widened) {
    *widened = false;
    if (sticky_sig.empty()) sticky_sig.assign(b->cols.size(), false);
    bool same = true;
    for (size_t i = 0; i < b->cols.size(); ++i) {
      const bool has = (bool)b->cols[i].validity;
      if (has && !sticky_sig[i]) { sticky_sig[i] = true; *widened = true; }
      same &= has == sticky_sig[i];
    }
    if (same) return b;
    const size_t need = (size_t)((b->rows + 31) / 32 * 4);
    if (!ones || ones_bytes < need) {
      ones_bytes = std::max<size_t>(need, 1 << 16);
      ones = dev_alloc(ctx, ones_bytes);
      SG_CUDA(cudaMemsetAsync(ones->ptr, 0xFF, ones_bytes, ctx->stream));
    }
    auto bb = std::make_shared<DevBatch>(*b);
    for (size_t i = 0; i < bb->cols.size(); ++i)
      if (sticky_sig[i] && !bb->cols[i].validity) { bb->cols[i].validity = ones; bb->cols[i].null_count = 0; }
    return bb;
  }

  static bool same_layout(const CompiledPipeline& a, const CompiledPipeline& b) {
    const AggParams &x = a.agg, &y = b.agg;
    if (x.entry_words != y.entry_words || x.key_words != y.key_words || x.has_null_word != y.has_null_word || x.n_accs != y.n_accs) return false;
    for (int j = 0; j < x.n_accs; ++j)
      if (x.accs[j].op != y.accs[j].op || x.accs[j].word != y.accs[j].word || x.accs[j].track_seen != y.accs[j].track_seen) return false;
    return a.acc_ident == b.acc_ident;
  }

  // the table built under `from`'s layout continues under `to`'s (a superset: more seen bits, a null-mask word, separate
  // counters where one counter served several aggregates)
  void migrate_layout(const std::shared_ptr<CompiledPipeline>& from, const std::shared_ptr<CompiledPipeline>& to) {
    Trace tr(ctx, "agg.migrate");
    const AggParams &O = from->agg, &N = to->agg;
    AggMigrateMap M;
    memset(&M, 0, sizeof(M));
    M.old_entry_words = (int32_t)O.entry_words; M.old_key_words = O.key_words;
    M.key_shift = (N.has_null_word && !O.has_null_word) ? 1 : 0;
    SG_CHECK(N.key_words == O.key_words + M.key_shift && N.has_null_word >= O.has_null_word, SAILGPU_ERR_UNSUPPORTED, "aggregate layouts of two batches cannot be reconciled (group keys)");
    std::vector<int> src((size_t)N.n_accs, -1);
    for (auto& kv : to->acc_ident) {
      auto it = from->acc_ident.find(kv.first);
      SG_CHECK(it != from->acc_ident.end(), SAILGPU_ERR_UNSUPPORTED, "aggregate layouts of two batches cannot be reconciled (" + kv.first + ")");
      src[(size_t)kv.second] = it->second;
    }
    for (int j = 0; j < N.n_accs; ++j) {
      SG_CHECK(src[(size_t)j] >= 0 && O.accs[src[(size_t)j]].op == N.accs[j].op, SAILGPU_ERR_UNSUPPORTED, "aggregate layouts of two batches cannot be reconciled (accumulator kinds)");
      M.acc_src_word[j] = (int16_t)O.accs[src[(size_t)j]].word;
      M.seen_src[j] = N.accs[j].track_seen ? (O.accs[src[(size_t)j]].track_seen ? (int8_t)src[(size_t)j] : (int8_t)-1) : (int8_t)-2;
    }
    const uint64_t groups = current_groups();
    AggTable old = tab;
    tab.table = dev_alloc(ctx, (size_t)tab.capacity * N.entry_words * 8);
    tab.state = dev_alloc_zero(ctx, (size_t)tab.capacity * 4);
    tab.occ = dev_alloc(ctx, (size_t)tab.capacity * 4);
    run.ensure_scratch();
    AggParams A = N;
    fill_table(A);
    SG_CUDA(cudaMemsetAsync(run.scal.n_groups(), 0, 8, ctx->stream));
    SG_CUDA(launch_agg_migrate(A, M, static_cast<const uint8_t*>(old.table->ptr), static_cast<const uint32_t*>(old.occ->ptr), groups, run.scal.error(), ctx->stream));
    m.kernel_launches++;
    known_groups = -1;
  }

  void push_agg(const BatchPtr& b0) {
    Trace tr(ctx, "agg.push");
    if (b0->rows == 0) return;
    bool widened = false;
    const BatchPtr b = with_union_signature(b0, &widened);
    auto cp = run.compiled_for(*b, use_cold);
    if (agg_cp && tab.capacity && !same_layout(*agg_cp, *cp)) {
      SG_CHECK(widened, SAILGPU_ERR_STATE, "aggregate layout changed without a new validity buffer");
      migrate_layout(agg_cp, cp);
    }
    agg_cp = cp;
    const bool grouped = cp->agg.n_keys > 0;
    // a pair set is bounded like a group table, so an aggregate with DISTINCT hands tiles back even without group keys
    const bool guarded = grouped || !cp->distinct.empty();
    if (dsets.empty() && !cp->distinct.empty()) {
      dsets.resize(cp->distinct.size());
      dcounts = dev_alloc_zero(ctx, MAX_DISTINCT * 8);
      const uint64_t cap = std::min<uint64_t>(std::min<uint64_t>(min_capacity(), max_capacity()), next_pow2(8 * (uint64_t)b->rows + 2048));
      for (size_t d = 0; d < dsets.size(); ++d) alloc_set(d, cp->distinct[d], cap, 0);
    }
    // first table: 4 M slots for real inputs, but a final aggregate over a few partial rows gets a few KB (a hand-back
    // grows it if later batches are bigger)
    if (!tab.capacity) alloc_table(cp->agg, grouped ? std::min<uint64_t>(std::min<uint64_t>(min_capacity(), max_capacity()), next_pow2(8 * (uint64_t)b->rows + 2048)) : 1024, 0);
    const int64_t tile_rows = (int64_t)cp->rpt * NT;
    const int64_t n_tiles = (b->rows + tile_rows - 1) / tile_rows;
    BufPtr deferred = guarded ? dev_alloc(ctx, (size_t)n_tiles * 4) : nullptr;
    const int slot = next_slot;
    launch_agg(cp, *b, nullptr, 0, deferred, slot);
    rows_in_table += b->rows;
    rows_seen_by_sets += b->rows;
    known_groups = -1;
    if (!guarded) return;
    next_slot ^= 1;
    copy_counters(slot, true);
    inflight.push_back({b, cp, deferred, slot});
    settle(1);
  }

  // Looks at the hand-back of every launch in flight but the newest `keep`.  With keep == 0 nothing is left in flight and
  // known_groups is the table's group count.
  void settle(size_t keep) {
    while (inflight.size() > keep) {
      const InFlight& f = inflight.front();
      const bool last = inflight.size() == 1;
      if (last) stream_sync(ctx);          // nothing else queued: this wait drains the stream
      else SG_CUDA(cudaEventSynchronize(copied[f.slot]));
      const Counters& c = counters[f.slot];
      if (c.error || c.n_def[f.slot]) { resolve_all(); return; }
      if (last) known_groups = (int64_t)c.n_groups;
      inflight.pop_front();
    }
  }

  int64_t rows_seen_by_sets = 0;      // rows pushed so far (rows_in_table restarts at a spill; the pair sets do not)

  // grows every pair set that is past its limit or, by the pairs per row seen so far, would be after the deferred rows
  void grow_sets(double rows_def) {
    if (dsets.empty()) return;
    std::vector<unsigned long long> pairs(dsets.size());
    SG_CUDA(cudaMemcpyAsync(pairs.data(), dcounts->ptr, pairs.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    const double rows_done = std::max(1.0, (double)rows_seen_by_sets - rows_def);
    const uint64_t ceiling = max_capacity();
    for (size_t d = 0; d < dsets.size(); ++d) {
      const uint64_t p = pairs[d];
      const double ratio = p ? std::min(1.0, (double)p / rows_done) : 1.0;
      uint64_t cap = next_pow2((uint64_t)(2.0 * ((double)p + ratio * rows_def * 1.25 + 1024.0)));
      const bool over = p > run.last_pair_limit[d];
      if (over && cap <= dsets[d].capacity) cap = dsets[d].capacity * 2;
      // the set is not partitioned: at the ceiling a set past its limit is refused before anything is allocated
      if (cap > ceiling) {
        SG_CHECK(!(over && dsets[d].capacity >= ceiling), SAILGPU_ERR_UNSUPPORTED, "count(DISTINCT) needs more than " + std::to_string(ceiling) + " pair slots");
        cap = ceiling;
      }
      if (cap > dsets[d].capacity) alloc_set(d, agg_cp->distinct[d], cap, p);
    }
  }

  // Slow path: some launch in flight handed tiles back or raised an error.  Drains the stream, then, until nothing is left,
  // grows the table for every deferred tile at once and re-launches over each list.
  void resolve_all() {
    Trace tr(ctx, "agg.resolve");
    stream_sync(ctx);
    const Counters* latest = &counters[inflight.back().slot];    // copied after the newest launch: the current values
    uint64_t prev_def = 0;
    const bool grouped = agg_cp->agg.n_keys > 0;
    for (;;) {
      raise_device_error(ctx, run.scal.error(), latest->error);
      const uint64_t groups = latest->n_groups;
      double rows_def = 0.0;
      uint64_t n_def_total = 0;
      for (auto& f : inflight) {
        const uint64_t n_def = latest->n_def[f.slot];
        n_def_total += n_def;
        rows_def += (double)std::min<int64_t>((int64_t)n_def * f.cp->rpt * NT, f.batch->rows);
      }
      if (n_def_total == 0) { known_groups = (int64_t)groups; break; }      // extract_agg() right after needs no second read-back
      const double rows_done = std::max(1.0, (double)rows_in_table - rows_def);
      // groups still to come, by the ratio seen so far (every row a new group when nothing was processed yet)
      const double ratio = groups ? std::min(1.0, (double)groups / rows_done) : 1.0;
      const double est = ratio * rows_def * 1.25 + 1024.0;
      uint64_t cap = next_pow2((uint64_t)(2.0 * ((double)groups + est)) + 2 * MIN_CAPACITY / 2);
      // a hand-back does not always mean a full table: the dictionary variant gives up at HOT_GROUP_LIMIT groups whatever the
      // capacity.  The table only grows when the estimate asks for it, or when a re-launch at this capacity made no progress.
      const bool stuck = prev_def != 0 && n_def_total >= prev_def;
      // (with pair sets a hand-back may have been for a set alone: then the group table does not double)
      if (cap <= tab.capacity && stuck && (dsets.empty() || groups > run.last_group_limit)) cap = tab.capacity * 2;
      prev_def = n_def_total;
      grow_sets(rows_def);
      // partitioned mode: the table grows to the ceiling and no further.  A full table at the ceiling hands its groups on as
      // state rows (spill) and starts over empty; the re-launches below then fill it again.
      const uint64_t ceiling = max_capacity();
      if (cap > ceiling && grouped) {
        cap = ceiling;
        if (tab.capacity >= ceiling && groups) {
          SG_CHECK(!partition_of_parent, SAILGPU_ERR_UNSUPPORTED, "a partition of a partitioned aggregate needs more than 2^28 group slots");
          spill(groups);
          rows_in_table = (int64_t)rows_def;
          prev_def = 0;
        }
      }
      if (cap > tab.capacity && grouped) alloc_table(inflight.front().cp->agg, cap, groups);
      if (!use_cold && groups > CARD_MANY_GROUPS) {
        auto cold = run.compiled_for(*inflight.front().batch, true);
        if (cold->agg.entry_words == inflight.front().cp->agg.entry_words) use_cold = true;     // later batches start on the many-groups variant
      }
      for (auto it = inflight.begin(); it != inflight.end();) {
        const uint64_t n_def = latest->n_def[it->slot];
        if (n_def == 0) { it = inflight.erase(it); continue; }
        if (use_cold && !it->cp->cold_variant) {
          auto cold = run.compiled_for(*it->batch, true);
          if (cold->rpt == it->cp->rpt && cold->agg.entry_words == it->cp->agg.entry_words) it->cp = cold;   // same tile size: the deferred list carries over
        }
        BufPtr next_deferred = dev_alloc(ctx, (size_t)n_def * 4);
        launch_agg(it->cp, *it->batch, it->deferred, (int64_t)n_def, next_deferred, it->slot);
        it->deferred = next_deferred;
        ++it;
      }
      const int slot = inflight.back().slot;
      copy_counters(slot, false);
      stream_sync(ctx);
      latest = &counters[slot];
    }
    inflight.clear();
  }

  // the table's group count with nothing in flight (error flag checked)
  uint64_t current_groups() {
    settle(0);
    if (known_groups < 0) {
      run.ensure_scratch();
      unsigned long long gd[4] = {0, 0, 0, 0};
      SG_CUDA(cudaMemcpyAsync(gd, run.scal.buf->ptr, 32, cudaMemcpyDeviceToHost, ctx->stream));      // error flag @0, n_groups @24
      stream_sync(ctx);
      raise_device_error(ctx, run.scal.error(), (uint32_t)gd[0]);
      known_groups = (int64_t)gd[3];
    }
    return (uint64_t)known_groups;
  }

  BatchPtr extract_agg() {
    Trace tr(ctx, "agg.extract");
    std::shared_ptr<CompiledPipeline> cp = agg_cp;
    if (!cp) {   // no input at all: compile against an all-valid signature to learn the output layout
      DevBatch dummy;
      for (auto& f : run.in_schema) { DevColumn c; c.type = f.type; dummy.cols.push_back(c); }
      cp = run.compiled_for(dummy);
    }
    run.ensure_scratch();
    const uint64_t groups = tab.capacity ? current_groups() : 0;
    return extract_rows(*cp, cp->agg_outs, groups);
  }

  // the table's `groups` groups as the columns `outs` describe (the operator's output, or the state rows of partitioned mode)
  BatchPtr extract_rows(const CompiledPipeline& cp, const std::vector<AggOutSpec>& outs, uint64_t groups) {
    const AggParams& A0 = cp.agg;
    run.ensure_scratch();
    const bool synth = A0.n_keys == 0 && groups == 0;   // global aggregate over zero rows: one row of NULLs / zero counts
    const int64_t rows = synth ? 1 : (int64_t)groups;
    auto out = std::make_shared<DevBatch>();
    out->rows = rows;
    AggExtractParams X;
    memset(&X, 0, sizeof(X));
    X.n_cols = (int)outs.size();
    std::vector<BufPtr> vbytes((size_t)X.n_cols);
    for (int i = 0; i < X.n_cols; ++i) {
      const AggOutSpec& s = outs[(size_t)i];
      AggOutCol& o = X.cols[i];
      o.kind = s.kind; o.a = s.a; o.b = s.b; o.c = s.c; o.var = s.var; o.nullable = s.nullable ? 1 : 0;
      o.width = s.type.is_string() ? 16 : s.type.arrow_width();
      SG_CHECK(s.type.id != TypeId::Bool, SAILGPU_ERR_UNSUPPORTED, "boolean group keys are not supported yet");
      if (s.kind == 0) { o.key_word = s.b; o.src_words = A0.keys[s.a].width == 16 ? 2 : 1; }
      else if (s.kind == 1) { const int op = A0.accs[s.a].op; o.src_words = (op == ACC_SUM_I128 || op == ACC_MIN_I128 || op == ACC_MAX_I128) ? 2 : 1; }
      else if (s.kind == 2) {
        o.is_float = s.type.is_float() ? 1 : 0;
        if (!o.is_float) { i128 mul = pow10_i128(s.type.scale - s.in_type.scale); o.scale_mul_lo = (uint64_t)(u128)mul; o.scale_mul_hi = (uint64_t)((u128)mul >> 64); }
      }
      DevColumn c; c.type = s.type; c.length = rows; c.arrow_is_utf8 = s.type.id == TypeId::Utf8;
      c.data = dev_alloc_zero(ctx, (size_t)rows * o.width);
      o.data = static_cast<uint8_t*>(c.data->ptr);
      if (s.nullable) { vbytes[(size_t)i] = dev_alloc_zero(ctx, (size_t)rows + 4); o.valid_bytes = static_cast<uint8_t*>(vbytes[(size_t)i]->ptr); }
      if (c.type.is_string()) c.heaps = kept_heaps;
      out->cols.push_back(c);
    }
    if (!synth && rows > 0) {
      AggParams A = A0;
      fill_table(A);
      SG_CUDA(launch_agg_extract(A, X, groups, run.scal.error(), ctx->stream));
      m.kernel_launches++;
    } else if (synth) {
      // counts are 0 (valid); every other aggregate is NULL -> validity bytes stay 0, count columns get no validity
      for (int i = 0; i < X.n_cols; ++i) {
        const AggOutSpec& s = outs[(size_t)i];
        const bool is_count = s.kind == 1 && (A0.accs[s.a].op == ACC_COUNT || (A0.accs[s.a].op == ACC_SUM_I64 && !A0.accs[s.a].track_seen));
        if (vbytes[(size_t)i] && is_count) SG_CUDA(cudaMemsetAsync(vbytes[(size_t)i]->ptr, 1, 1, ctx->stream));
      }
    }
    // Outputs that cannot be null under this layout (keys without a null word, sums whose inputs carry no validity) have no
    // validity to pack; only when some output can be null are the null counts read back, so that an all-valid bitmap is dropped
    bool any_nullable = false;
    for (int i = 0; i < X.n_cols; ++i) any_nullable |= vbytes[(size_t)i] && rows > 0;
    if (!any_nullable) return out;
    std::vector<unsigned long long> nulls((size_t)X.n_cols, 0);
    BufPtr nullctr = dev_alloc_zero(ctx, (size_t)X.n_cols * 8 + 8);
    for (int i = 0; i < X.n_cols; ++i) {
      if (!vbytes[(size_t)i] || rows == 0) continue;
      DevColumn& c = out->cols[(size_t)i];
      c.validity = dev_alloc_zero(ctx, (size_t)((rows + 31) / 32 * 4));
      SG_CUDA(launch_pack_bytes(static_cast<const uint8_t*>(vbytes[(size_t)i]->ptr), static_cast<uint32_t*>(c.validity->ptr), rows,
                                static_cast<unsigned long long*>(nullctr->ptr) + i, ctx->stream));
    }
    SG_CUDA(cudaMemcpyAsync(nulls.data(), nullctr->ptr, (size_t)X.n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
    // the extraction raises an overflow for avg(Decimal) (every such output is nullable, so this read-back covers it)
    uint32_t err = 0;
    SG_CUDA(cudaMemcpyAsync(&err, run.scal.error(), 4, cudaMemcpyDeviceToHost, ctx->stream));
    stream_sync(ctx);
    raise_device_error(ctx, run.scal.error(), err);
    for (int i = 0; i < X.n_cols; ++i) {
      DevColumn& c = out->cols[(size_t)i];
      if (c.validity) { c.null_count = (int64_t)nulls[(size_t)i]; if (c.null_count == 0) c.validity = nullptr; }
    }
    return out;
  }

  // ---- partitioned mode ------------------------------------------------------------------------
  // A table at the ceiling (max_capacity) that would have to grow hands its groups on as partial-aggregate state rows and
  // starts over.  A partial aggregate emits those rows right away (the final aggregate after it merges a group emitted more
  // than once).  The other modes keep them in HBM; when the input has ended, the rows still in the table join them, they
  // are hash-partitioned on the group key by RepartitionOp, and one final aggregate per partition merges each partition's
  // rows in a table of its own.  Aggregates whose table stays under the ceiling never get here.
  std::vector<BatchPtr> spilled;

  // State rows as a partial aggregate emits them: keys, then each aggregate's state columns.  Every mode's table holds the
  // accumulators of those states (compiler.cu finish_aggregate: single and partial compile the same accumulators, the final
  // modes merge state columns into accumulators of the same kinds, avg as a count and a sum, Decimal128 sums in 128 bits);
  // only the outputs differ, where avg is sum / count and the variance family's count, mean and m2 become one value.
  static std::vector<AggOutSpec> state_outs(const CompiledPipeline& cp) {
    std::vector<AggOutSpec> outs;
    for (const AggOutSpec& s : cp.agg_outs) {
      if (s.kind == 5) {
        AggOutSpec c = s, mean = s, m2 = s;
        c.kind = 1; c.a = s.b; c.b = 0; c.type = T(TypeId::UInt64); c.nullable = false;
        mean.kind = 3; mean.a = s.c; mean.nullable = false;
        m2.kind = 4; m2.nullable = false;
        outs.push_back(c); outs.push_back(mean); outs.push_back(m2);
        continue;
      }
      if (s.kind != 2) { outs.push_back(s); continue; }
      AggOutSpec c = s, v = s;
      c.kind = 1; c.a = s.b; c.b = 0; c.type = T(TypeId::UInt64); c.nullable = false;
      v.kind = 1; v.b = 0; v.type = agg_types("avg", s.in_type).state[1]; v.nullable = cp.agg.accs[s.a].track_seen != 0;
      outs.push_back(c); outs.push_back(v);
    }
    return outs;
  }

  void spill(uint64_t groups) {
    Trace tr(ctx, "agg.spill");
    BatchPtr rows = extract_rows(*agg_cp, state_outs(*agg_cp), groups);
    SG_CUDA(cudaMemsetAsync(tab.state->ptr, 0, (size_t)tab.capacity * 4, ctx->stream));
    SG_CUDA(cudaMemsetAsync(run.scal.n_groups(), 0, 8, ctx->stream));
    known_groups = -1;
    m.agg_spills++;
    if (run.stages.back().mode == "partial") ready.push_back(rows);
    else spilled.push_back(rows);
  }

  static Json jnum(int64_t v) { Json j; j.kind = Json::Num; j.s = std::to_string(v); return j; }
  static Json jstr(const std::string& v) { Json j; j.kind = Json::Str; j.s = v; return j; }
  static Json jcol(int64_t i) { Json j; j.kind = Json::Obj; j.o = {{"col", jnum(i)}}; return j; }

  // the end of the input in partitioned mode (single / final / final_partitioned): one output batch per partition
  void finish_partitioned() {
    Trace tr(ctx, "agg.partitions");
    const std::shared_ptr<CompiledPipeline> cp = agg_cp;
    const uint64_t left = current_groups();
    if (left) spilled.push_back(extract_rows(*cp, state_outs(*cp), left));
    const StageSpec& st = run.stages.back();
    const int n_keys = (int)st.group_exprs.size();
    Schema states;
    const std::vector<AggOutSpec> souts = state_outs(*cp);
    for (size_t i = 0; i < souts.size(); ++i)
      states.push_back({i < (size_t)n_keys ? out_schema[i].name : "__state" + std::to_string(i), souts[i].type, souts[i].nullable || (i < (size_t)n_keys && out_schema[i].nullable)});
    uint64_t rows = 0;
    for (auto& b : spilled) rows += (uint64_t)b->rows;
    // P: the smallest power of two that leaves at most an eighth of the ceiling's slots in state rows per partition.  A
    // partition's rows bound its groups, so its table ends at most a quarter full and never reaches the ceiling itself.
    const uint64_t per_part = std::max<uint64_t>(1, max_capacity() / 8);
    uint64_t n_parts = 1;
    while (n_parts * per_part < rows) n_parts *= 2;
    SG_CHECK(n_parts <= 4096, SAILGPU_ERR_UNSUPPORTED, "aggregate needs more than 4096 key-hash partitions");
    std::vector<std::vector<BatchPtr>> parts((size_t)n_parts);
    if (n_parts == 1) parts[0].swap(spilled);
    else {
      // the partition of a row is RepartitionOp's hash of the key values (nulls and string contents, not views) modulo P: the
      // low bits of a hash that the group table's probe (pipeline.cu hash_packed_key: another seed, another mixing chain) does
      // not share, so every partition's keys still spread over all slots of its table
      Json keys; keys.kind = Json::Arr;
      for (int i = 0; i < n_keys; ++i) keys.a.push_back(jcol(i));
      Json spec; spec.kind = Json::Obj;
      spec.o = {{"op", jstr("repartition")}, {"scheme", jstr("hash")}, {"exprs", keys}, {"n", jnum((int64_t)n_parts)}};
      std::unique_ptr<Op> rp = make_op(ctx, spec, {states}, 0);
      for (auto& b : spilled) rp->push(0, b);
      spilled.clear();
      rp->finish(0);
      for (uint64_t p = 0; p < n_parts; ++p)
        for (;;) { BatchPtr b; const bool more = rp->pull_partition((int)p, &b); if (b && b->rows) parts[(size_t)p].push_back(b); if (!more) break; }
      m.kernel_launches += rp->m.kernel_launches;
    }
    // one final aggregate per partition over the state rows: [keys | states] -> the operator's output.  A DISTINCT aggregate
    // merges as its plain counterpart (no "distinct" here): the pair sets were never emptied, so each pair was counted in
    // exactly one state row, and a sum of counts / sums over the state rows is the DISTINCT result.
    Json gb; gb.kind = Json::Arr;
    for (int i = 0; i < n_keys; ++i) { Json g; g.kind = Json::Obj; g.o = {{"expr", jcol(i)}, {"name", jstr(st.group_names[(size_t)i])}}; gb.a.push_back(g); }
    Json aggs; aggs.kind = Json::Arr;
    for (auto& a : st.aggs) {
      Json j; j.kind = Json::Obj;
      j.o = {{"fn", jstr(a.fn)}, {"name", jstr(a.name)}};
      if (a.input_type.id != TypeId::Null) j.o.push_back({"input_type", jstr(a.input_type.str())});
      aggs.a.push_back(j);
    }
    Json fspec; fspec.kind = Json::Obj;
    fspec.o = {{"op", jstr("aggregate")}, {"mode", jstr("final")}, {"group_by", gb}, {"aggs", aggs}};
    m.agg_partition_groups.assign((size_t)n_parts, 0);
    for (uint64_t p = 0; p < n_parts; ++p) {
      std::vector<BatchPtr> in;
      in.swap(parts[(size_t)p]);
      if (in.empty()) continue;
      std::unique_ptr<Op> op = make_op(ctx, fspec, {states}, 0);
      PipelineOp* po = dynamic_cast<PipelineOp*>(op.get());
      SG_CHECK(po != nullptr, SAILGPU_ERR_STATE, "partitioned aggregate: the per-partition aggregate is not a hash aggregate");
      po->partition_of_parent = true;
      for (auto& b : in) op->push(0, b);
      in.clear();
      op->finish(0);
      std::vector<BatchPtr> outs;
      for (;;) { BatchPtr o; const bool more = op->pull(&o); if (o && o->rows) outs.push_back(o); if (!more) break; }
      m.kernel_launches += op->m.kernel_launches;
      if (outs.empty()) continue;
      BatchPtr o = outs.size() == 1 ? outs[0] : concat_batches(ctx, out_schema, outs);
      m.agg_partition_groups[(size_t)p] = (uint64_t)o->rows;
      ready.push_back(o);
    }
    m.agg_partitions = n_parts;
    if (ready.empty()) ready.push_back(empty_batch(ctx, out_schema));
  }
};

// Plan-time specialisation (sailgpu_jit_precompile): compiles the pipeline of `spec` for a batch whose columns carry
// validity buffers where `validity_mask` has a bit set, writes the specialised kernel's source to *source and, with
// `compile`, its cubin into the kernel cache -- all without a device (NVRTC cross-compiles for sm_90a).
size_t pipeline_precompile(const Json& spec, const std::vector<Schema>& inputs, uint64_t validity_mask, bool cold, bool compile, std::string* source) {
  static Ctx plan_ctx;      // H100 geometry (132 SMs, 227 KB of shared memory per CTA); never touches a device
  std::unique_ptr<Op> op = make_op(&plan_ctx, spec, inputs, 0);
  PipelineOp* p = dynamic_cast<PipelineOp*>(op.get());
  SG_CHECK(p != nullptr, SAILGPU_ERR_UNSUPPORTED, "only filter / projection / aggregate pipelines are specialised");
  DevBatch shape;
  for (size_t i = 0; i < inputs[0].size(); ++i) {
    DevColumn c; c.type = inputs[0][i].type;
    if (i < 64 && ((validity_mask >> i) & 1)) c.validity = std::make_shared<DevBuf>();
    shape.cols.push_back(c);
  }
  auto cp = p->run.compiled_for(shape, cold);
  std::string why;
  SG_CHECK(jit_supported(*cp, &why), SAILGPU_ERR_UNSUPPORTED, "kernel specialiser: " + why);
  JitPlan plan;
  SG_CHECK(jit_plan(*cp, plan_ctx.max_smem, &plan), SAILGPU_ERR_UNSUPPORTED, "kernel specialiser: pipeline does not fit in shared memory");
  const std::string src = jit_generate(*cp, plan);
  if (source) *source = src;
  return compile ? jit_precompile_to_cache(src) : 0;
}

// Plan-time limits of a filter / projection / aggregate pipeline (sailgpu_spec_validate): the tile program is compiled against the
// H100 geometry for a batch without validity buffers, so that the data-independent limits -- "more than 6 group keys", "group key
// wider than 64 bytes", "does not fit in shared memory" ... -- are answered while planning, never after the first batch arrived.
// (Validity buffers add one column buffer each; a batch whose nullable columns push a pipeline over the 20-buffer limit is still
// reported at push time as SAILGPU_ERR_UNSUPPORTED.)  Touches no device.
static thread_local bool g_in_static_check = false;
std::unique_ptr<Op> make_wide_agg_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs, const Schema& out_schema);
void pipeline_static_check(const Json& spec, const std::vector<Schema>& inputs) {
  static Ctx plan_ctx;
  std::unique_ptr<Op> op = make_op(&plan_ctx, spec, inputs, 0);
  PipelineOp* p = dynamic_cast<PipelineOp*>(op.get());
  if (p == nullptr || p->rename_only()) return;       // a projection that only picks / renames columns passes buffers on: nothing to compile
  DevBatch shape;
  for (auto& f : inputs[0]) { DevColumn c; c.type = f.type; shape.cols.push_back(c); }
  p->run.compiled_for(shape, false);
}

std::unique_ptr<Op> make_join_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs);
std::unique_ptr<Op> make_sort_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs);
std::unique_ptr<Op> make_merge_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs);
std::unique_ptr<Op> make_nlj_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs);
std::unique_ptr<Op> make_repartition_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs);
std::unique_ptr<Op> make_chain_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs);
std::unique_ptr<Op> make_exchange_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs);

std::unique_ptr<Op> make_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs, int partition) {
  (void)partition;
  const std::string kind = spec.at("op").as_str();
  if (kind == "hash_join") return make_join_op(ctx, spec, inputs);
  if (kind == "nested_loop_join") return make_nlj_op(ctx, spec, inputs);
  if (kind == "sort") return make_sort_op(ctx, spec, inputs);
  if (kind == "sort_preserving_merge") return make_merge_op(ctx, spec, inputs);
  if (kind == "repartition") return make_repartition_op(ctx, spec, inputs);
  if (kind == "chain") return make_chain_op(ctx, spec, inputs);
  if (kind == "exchange") return make_exchange_op(ctx, spec, inputs);
  SG_CHECK(inputs.size() == 1, SAILGPU_ERR_INVALID, "operator '" + kind + "' takes exactly one input");
  auto op = std::make_unique<PipelineOp>();
  op->ctx = ctx; op->kind = kind; op->in_schemas = inputs;
  op->run.init(ctx, inputs[0]);
  std::vector<const Json*> stage_specs;
  if (kind == "pipeline") for (auto& s : spec.at("stages").a) stage_specs.push_back(&s);
  else stage_specs.push_back(&spec);
  SG_CHECK(!stage_specs.empty(), SAILGPU_ERR_INVALID, "empty pipeline");
  Schema cur = inputs[0];
  for (const Json* s : stage_specs) {
    Schema next;
    op->run.stages.push_back(parse_stage(*s, cur, &next));
    cur = next;
  }
  {   // operators created from the same spec over the same schema share their compiled pipelines (and specialised kernels)
    std::string key = "pipeline|";
    json_dump(spec, &key);
    for (auto& f : inputs[0]) { key += '|'; key += f.type.str(); key += f.nullable ? '?' : '!'; }
    op->share_key = key;
    op->run.share(key);
  }
  op->has_agg = op->run.stages.back().kind == StageSpec::Aggregate;
  for (size_t i = 0; i + 1 < op->run.stages.size(); ++i)
    SG_CHECK(op->run.stages[i].kind != StageSpec::Aggregate, SAILGPU_ERR_INVALID, "aggregate must be the last stage of a pipeline");
  op->out_schema = cur;
  // a group key the hash table cannot pack (more than 6 keys / 64 bytes): grouping by sorting instead (ops_more.cu WideAggOp)
  // The verdict depends on the spec and the input schema only: it is kept with the operator's compiled pipelines, so that
  // re-creating the same plan (every execution of a query) compiles nothing on the host.
  if (kind == "aggregate" && !g_in_static_check) {
    std::shared_ptr<bool> verdict;
    const std::string vkey = "wide_agg|" + op->share_key;
    const bool cacheable = ctx && ctx->stream != nullptr;
    if (cacheable) {
      auto it = ctx->shared_objects.find(vkey);
      if (it != ctx->shared_objects.end()) verdict = std::static_pointer_cast<bool>(it->second);
    }
    if (!verdict) {
      bool wide = false;
      g_in_static_check = true;
      try { pipeline_static_check(spec, inputs); }
      catch (const Error& e) { wide = e.code == SAILGPU_ERR_UNSUPPORTED && std::string(e.what()).find("group key") != std::string::npos; }
      g_in_static_check = false;
      verdict = std::make_shared<bool>(wide);
      if (cacheable) ctx->shared_objects.emplace(vkey, std::static_pointer_cast<void>(verdict));
    }
    if (*verdict) return make_wide_agg_op(ctx, spec, inputs, cur);
  }
  return op;
}

}  // namespace sg
