//! sail-gpu -- H100 execution of Sail's physical-plan hot path behind DataFusion's `ExecutionPlan`.
//!
//! NOT COMPILED in this repository (the build image has no Rust toolchain); see shim/README.md.
//!
//! * `ffi`     -- the `extern "C"` surface of include/sailgpu.h, one binding per entry point
//! * `spec`    -- DataFusion physical nodes / expressions -> the JSON operator specs libsailgpu takes
//! * `exec`    -- `GpuExec`: an `ExecutionPlan` whose stream pushes child batches into a `sailgpu_op` and pulls results
//! * `rewrite` -- the pass `LocalJobRunner::execute` / `TaskRunner::execute_plan` call before `trace_execution_plan`
//! * `config`  -- the `execution.gpu.*` keys (crates/sail-common/src/config/application.yaml)
pub mod config;
pub mod exec;
pub mod ffi;
pub mod rewrite;
pub mod spec;

pub use config::GpuOptions;
pub use exec::GpuExec;
pub use rewrite::rewrite_for_gpu;
