// jit.hpp -- pipeline specialiser: CompiledPipeline -> CUDA source -> NVRTC (sm_90a) -> loaded kernel.
#pragma once
#include <string>

#include "compiler.hpp"

namespace sg {

constexpr size_t JIT_HDR_BYTES = 256;     // shared-memory header of a specialised kernel (jit_rt.cuh: JIT_HDR)

struct JitKernel {
  void* module = nullptr;      // CUmodule
  void* func = nullptr;        // CUfunction
  int rpt = 0, stages = 0, minb = 0;
  size_t smem_bytes = 0;
  int ctas_per_sm = 0;
  std::string key;
};

struct JitPlan {       // geometry chosen by the host for one pipeline
  int rpt = 2, stages = 2, minb = 2;
  uint32_t stage_bytes = 0, scratch_bytes = 0;
  size_t smem_bytes = 0;
};

// false: this pipeline is not covered by the specialiser (stays on the interpreter); *why says which construct
bool jit_supported(const CompiledPipeline& cp, std::string* why);
// geometry for `cp` at the interpreter's tile size (cp.rpt); false when nothing fits
bool jit_plan(const CompiledPipeline& cp, size_t max_smem, JitPlan* plan);
// CUDA source of the specialised kernel (host only: needs no device)
std::string jit_generate(const CompiledPipeline& cp, const JitPlan& plan);
// NVRTC-compiles `source` for sm_90a; returns the cubin bytes or throws sg::Error with the compiler log
std::string jit_compile_cubin(const std::string& source);
// cached (memory, then <lib dir>/jit_cache) compile + load; needs a current CUDA context
std::shared_ptr<JitKernel> jit_get_kernel(const CompiledPipeline& cp, size_t max_smem);
// launch through the driver API
void jit_launch(const JitKernel& k, const KernelArgs& K, int grid, cudaStream_t stream);
// mode from SAILGPU_JIT: 0 off, 1 on (default)
bool jit_enabled();
// rows an operator must have seen before a pipeline is worth compiling (SAILGPU_JIT_MIN_ROWS; cached kernels are used at once)
int64_t jit_min_rows();
bool jit_cached(const CompiledPipeline& cp, size_t max_smem);
// compiles `source` into the on-disk kernel cache unless it is there already; returns the cubin size (no device needed)
size_t jit_precompile_to_cache(const std::string& source);

}  // namespace sg
