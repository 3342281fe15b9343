// engine.hpp -- operator objects behind the C ABI (one per DataFusion operator instance+partition).
#pragma once
#include <chrono>
#include <deque>

#include "compiler.hpp"
#include "device.hpp"
#include "kernels.hpp"

namespace sg {

BatchPtr take_internal_batch(ArrowDeviceArray* arr, Ctx* consumer);   // device.cu

struct Metrics {
  uint64_t input_rows = 0, input_batches = 0, output_rows = 0, output_batches = 0;
  uint64_t elapsed_compute_ns = 0, kernel_launches = 0;
  uint64_t build_input_rows = 0, build_input_batches = 0, build_time_ns = 0, join_time_ns = 0;
  uint64_t pipeline_launches = 0, pipeline_kernel_ns = 0, jit_launches = 0;
  uint64_t host_syncs = 0;      // stream drains during calls on this operator's handle (import and export included), capi.cu
  // partitioned mode of a hash aggregate (engine.cu): times the table was emptied at its ceiling, key-hash partitions, groups
  // each partition's final aggregate produced
  uint64_t agg_spills = 0, agg_partitions = 0;
  std::vector<uint64_t> agg_partition_groups;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;   // CUDA events bracketing each pipeline-kernel launch
};

struct Op {
  Ctx* ctx = nullptr;
  std::vector<Schema> in_schemas;
  Schema out_schema;
  std::string last_error;
  std::string kind;
  Metrics m;
  virtual ~Op() { if (!g_exiting.load()) for (auto& p : m.pending) { cudaEventDestroy(p.first); cudaEventDestroy(p.second); } }
  // device time spent inside pipeline_kernel launches (resolves the pending event pairs; synchronises them)
  uint64_t pipeline_kernel_ns() {
    for (auto& p : m.pending) {
      float ms = 0.f;
      if (cudaEventSynchronize(p.second) == cudaSuccess && cudaEventElapsedTime(&ms, p.first, p.second) == cudaSuccess)
        m.pipeline_kernel_ns += (uint64_t)((double)ms * 1e6);
      cudaEventDestroy(p.first); cudaEventDestroy(p.second);
    }
    m.pending.clear();
    return m.pipeline_kernel_ns;
  }
  virtual void push(int input, const BatchPtr& b) = 0;
  virtual void finish(int input) = 0;
  // returns has_more; *out == nullptr when nothing is ready yet
  virtual bool pull(BatchPtr* out) = 0;
  virtual bool pull_partition(int, BatchPtr*) { fail(SAILGPU_ERR_STATE, "operator has no partitioned output"); }
};

std::unique_ptr<Op> make_op(Ctx* ctx, const Json& spec, const std::vector<Schema>& inputs, int partition);

// shared helpers (engine.cu)
StageSpec parse_stage(const Json& j, const Schema& in, Schema* out);
void check_device_error(Ctx* ctx, uint32_t* dev_flag);

// Small device scratch shared by every launch of an op: error flag, counters.
struct DevScalars {
  BufPtr buf;     // [0] u32 error flag, [8] u64 out_count, [16] u32 ticket, [24] u64 n_groups, [32] u64 cursor, [40] u64 null counters[...]
  uint32_t* error() const { return reinterpret_cast<uint32_t*>(buf->ptr); }
  unsigned long long* out_count() const { return reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(buf->ptr) + 8); }
  unsigned int* ticket() const { return reinterpret_cast<unsigned int*>(static_cast<uint8_t*>(buf->ptr) + 16); }
  unsigned long long* n_groups() const { return reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(buf->ptr) + 24); }
  unsigned long long* cursor() const { return reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(buf->ptr) + 32); }
  unsigned long long* nulls(int i) const { return reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(buf->ptr) + 64 + 8 * i); }
};

}  // namespace sg
