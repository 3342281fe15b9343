/*
 * sailgpu.h -- C ABI of libsailgpu.so: the H100-native replacement for the DataFusion physical
 * operators on Sail's hot path.
 *
 * Who binds this.  A Rust shim crate inside Sail (see INTEGRATION.md) implements
 * `datafusion::physical_plan::ExecutionPlan` once per replaced operator and drives this API from
 * the `SendableRecordBatchStream` it returns from `execute(partition, ctx)`:
 *
 *   reference interface this replaces (file:line under lakehq/sail)         entry points here
 *   ---------------------------------------------------------------------   ---------------------------
 *   ExecutionPlan::execute(partition, Arc<TaskContext>)                      sailgpu_op_create
 *     crates/sail-execution/src/plan/shuffle_write.rs:146-206 (shape),
 *     crates/sail-physical-plan/src/streaming/filter.rs:104-116
 *   RecordBatchStream::poll_next: pull child batch, hand it to the operator  sailgpu_op_push[_device],
 *     crates/sail-execution/src/plan/shuffle_write.rs:226-232                sailgpu_op_finish_input
 *   RecordBatchStream::poll_next: yield Result<RecordBatch>                  sailgpu_op_pull[_device]
 *   RecordBatchStream::schema() / ExecutionPlan::schema()                    out_schema of op_create
 *   ExecutionPlan::metrics() (names in crates/sail-telemetry/src/execution/  sailgpu_op_metrics
 *     metrics/{default,filter,join,projection}.rs)
 *   drop(stream) == cancellation (repartition.rs:104-119)                    sailgpu_op_destroy
 *   DataFusionError travelling as a stream item (stream/error.rs:38-70)      int32 status +
 *                                                                            sailgpu_last_error
 *   LocalJobRunner::execute / TaskRunner::execute_plan rewrite hook          (shim side; no C call)
 *     crates/sail-execution/src/job_runner.rs:63, task_runner/core.rs:110
 *   shuffle_write / shuffle_read for Partitioning::Hash                      op kind "repartition" +
 *     crates/sail-execution/src/plan/shuffle_write.rs:209-267,               sailgpu_ctx_comm_init,
 *     plan/shuffle_read.rs:107-117                                           sailgpu_exchange
 *
 * Data crosses the boundary as Arrow C Data Interface structs (host memory, pageable is fine: packer
 * threads of the library range-check every column piece, write it in a narrow wire format into pinned
 * staging memory and expand it back to Arrow in HBM, sail_b200/csrc/h2d.cu) or Arrow C *Device* Data Interface structs
 * (ARROW_DEVICE_CUDA: buffers already in HBM, zero copy -- how consecutive GPU operators chain
 * without bouncing through the host).  No torch types, no C++ types: plain pointers and sizes.
 *
 * Operator specs are small JSON documents (UTF-8) mirroring DataFusion's plan-node fields:
 *   {"op":"filter","predicate":E,"projection":[i,...]|null}
 *   {"op":"projection","exprs":[{"expr":E,"name":"..."},...]}
 *   {"op":"aggregate","mode":"partial|final|final_partitioned|single",
 *    "group_by":[{"expr":E,"name":".."}],"aggs":[{"fn":"sum|avg|count|min|max|stddev|stddev_pop|var|var_pop","args":[E],
 *    "name":"..","input_type":"T","distinct":false|true}]}
 *                                          ("distinct": true -- count / sum / avg(DISTINCT E) -- in mode single only, over one
 *                                           argument that is not Float32 / Float64 / Boolean, at most 4 distinct arguments per
 *                                           aggregate; for min / max the flag is a no-op)
 *                                          (stddev / var: the sample forms, stddev_pop / var_pop: the population forms, under
 *                                           DataFusion's physical names; aliases such as variance or stddev_samp are refused.
 *                                           The argument is any integer, Decimal128, Float32 or Float64, converted to Float64;
 *                                           the result is Float64, NULL below 2 (sample) or 1 (population) non-null values.
 *                                           Partial state: name[count] UInt64, name[mean] Float64, name[m2] Float64 (sum of
 *                                           squared deviations; 0, 0.0, 0.0 for a group without values).  Sums are kept in
 *                                           double-double, so results stay within about 1e-10 relative even where |mean| / stddev
 *                                           is 1e8; equal values give exactly 0.0.  A group holding NaN or +-inf gives NaN, a
 *                                           single one included (DataFusion's ungrouped accumulator reports 0.0 for var_pop of
 *                                           one non-finite value), and so does a value whose square leaves Float64 (|x| above
 *                                           about 1.3e154); the partial mean and m2 of such a group are NaN.)
 *   {"op":"hash_join","join_type":"inner|left|right|left_semi|left_anti|right_semi|right_anti","on":[[l,r],...],
 *    "filter":E|null,"projection":[...]|null}   (input 0 = build = LEFT child, input 1 = probe; residual filters with
 *                                           inner, right_semi, left_semi and left_anti)
 *   {"op":"nested_loop_join","join_type":"inner","filter":E|null,"projection":[...]|null}
 *                                          (NestedLoopJoinExec with a small build side: the scalar-subquery shapes)
 *   {"op":"sort","keys":[{"expr":E,"asc":bool,"nulls_first":bool}],"fetch":k|null}     (fetch: TopK by radix selection)
 *   {"op":"sort_preserving_merge","keys":[...],"fetch":k|null,"runs":"inputs|batches"}
 *                                          (SortPreservingMergeExec: one input per sorted partition, k-way merge)
 *   {"op":"repartition","scheme":"hash","exprs":[E],"n":N}
 *   {"op":"repartition","scheme":"round_robin_row","n":N,"input_partition":i,"num_input_partitions":m}
 *                                          (RowRoundRobinPartitioner of ExplicitRepartitionExec, repartition.rs:46-84)
 *   {"op":"pipeline","stages":[spec,...]}  (fused chain of filter/projection ending in at most one
 *                                           aggregate: one kernel, one pass over HBM)
 *   {"op":"chain","ops":[spec,...]}        (consecutive single-input operators run as one GPU island:
 *                                           batches move between them inside the library, in HBM)
 *   {"op":"exchange","mode":"hash|gather|auto","exprs":[E],"root":r,"small_rows":k,"keep_runs":bool}
 *                                          (the shuffle boundary inside a chain: hash-repartition + NCCL
 *                                           all-to-all, or coalesce on rank r; needs sailgpu_ctx_comm_init)
 * Expressions E: {"col":i} {"lit":v,"type":"T"} {"op":"+|-|*|/|%|=|!=|<|<=|>|>=|and|or","l":E,"r":E}
 *   {"not":E} {"neg":E} {"is_null":E} {"is_not_null":E} {"cast":E,"to":"T"}
 *   {"case":[[E,E],...],"else":E|null} {"in":E,"set":[lit,...],"negated":b}
 *   {"like":E,"pattern":"..","negated":b} {"fn":"date_part","part":"year|month|day","args":[E]}   (E Date32)
 *   {"fn":"date_part","part":"year|quarter|month|day|hour|minute|second","args":[E]}   (E Timestamp: Int32, second as
 *                                           Decimal128(8,6), the microsecond within the minute; in the column's zone)
 *   {"fn":"date_trunc","part":"year|quarter|month|week|day|hour|minute|second","args":[E]}   (E Timestamp -> its type)
 *   {"fn":"substr","args":[E],"start":s,"length":n|null}   (1-based, in characters)
 *   {"fn":"character_length","args":[E]}   (E Utf8 / Utf8View -> Int32: the bytes that are not UTF-8 continuation bytes,
 *                                           i.e. the characters of valid UTF-8; NULL for NULL)
 * Types T: Boolean Int8..Int64 UInt8..UInt64 Float32 Float64 Date32 Decimal128(p,s) Utf8 Utf8View
 *   Timestamp(s|ms|us|ns[, zone]) (Arrow tss: / tsm: / tsu: / tsn: + zone; stored as Int64).  Any zone passes through the
 *   operators; date_part, date_trunc and the cast to Date32 read wall-clock time and accept no zone, UTC or +HH:MM / -HH:MM
 *   only (other zones: SAILGPU_ERR_UNSUPPORTED).  Casts: Int64 <-> Timestamp (same value), Timestamp -> Date32, Timestamp ->
 *   Timestamp of the same or a finer unit; comparisons between timestamps of one unit; no arithmetic, sum or avg.
 *   Range: the calendar parts and truncations (year .. day, week) and the cast to Date32 count days in 32 bits, so they are exact
 *   for instants within about 5.8 million years of the epoch (Date32's range) and wrong beyond it, which only Timestamp(s) and
 *   Timestamp(ms) can reach; the cast to a finer unit wraps when the product leaves int64 (arrow-rs reports an error there).
 *
 * Threading (SURVEY.md section 8b): any function may be called from any thread (no affinity: the
 * device is set per call); calls on one handle must not overlap.  A context owns ONE compute stream,
 * allocation cache and D2H staging block, so calls on handles of the same context are serialised
 * inside the library (they are correct from any number of threads, they do not overlap on the GPU);
 * partitions that should run concurrently use one context each -- contexts share nothing.
 * There is NO CPU fallback: every function fails with SAILGPU_ERR_NO_DEVICE if CUDA is unusable.
 */
#ifndef SAILGPU_H
#define SAILGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Arrow C Data Interface (https://arrow.apache.org/docs/format/CDataInterface.html) ---- */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4
struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};
struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif

/* ---- Arrow C Device Data Interface ---- */
#ifndef ARROW_C_DEVICE_DATA_INTERFACE
#define ARROW_C_DEVICE_DATA_INTERFACE
typedef int32_t ArrowDeviceType;
#define ARROW_DEVICE_CPU 1
#define ARROW_DEVICE_CUDA 2
#define ARROW_DEVICE_CUDA_HOST 3
struct ArrowDeviceArray {
  struct ArrowArray array;   /* buffer pointers are device pointers */
  int64_t device_id;
  ArrowDeviceType device_type;
  void* sync_event;          /* cudaEvent_t* or NULL */
  int64_t reserved[3];
};
#endif

#if defined(__GNUC__)
#define SAILGPU_API __attribute__((visibility("default")))
#else
#define SAILGPU_API
#endif

typedef struct sailgpu_ctx sailgpu_ctx; /* per process+device: stream pool, HBM pool, pinned staging, NCCL comm */
typedef struct sailgpu_op sailgpu_op;   /* one operator instance for one partition */

enum {
  SAILGPU_OK = 0,
  SAILGPU_ERR_INVALID = 1,      /* bad argument / malformed spec            -> DataFusionError::Plan      */
  SAILGPU_ERR_UNSUPPORTED = 2,  /* type/expression not implemented on GPU   -> DataFusionError::NotImplemented */
  SAILGPU_ERR_CUDA = 3,         /* CUDA / NCCL runtime failure              -> DataFusionError::Execution */
  SAILGPU_ERR_ARITHMETIC = 4,   /* checked arithmetic failed on a row that is evaluated -> ArrowError::DivideByZero / ArithmeticOverflow:
                                   integer or decimal `/` `%` by zero; integer MIN / -1 and MIN % -1; a decimal `/` `%` whose operand,
                                   rescaled to the division's scale, leaves i128; avg(Decimal) whose sum * 10^(s_out - s_in) leaves i128.
                                   `+` `-` `*` and sum() wrap (Int mod 2^64, Decimal128 mod 2^128), as DataFusion's default
                                   fail_on_overflow = false does, and raise nothing */
  SAILGPU_ERR_NO_DEVICE = 5,    /* no usable CUDA device: there is no CPU fallback */
  SAILGPU_ERR_STATE = 6         /* call sequence violation (push after finish, ...) -> DataFusionError::Internal */
};

/* Release callback for a borrowed copy of an ArrowArray struct (shares the producer's buffers, owns nothing): lets one
 * HBM-resident batch be pushed into several operators. */
SAILGPU_API void sailgpu_borrowed_release(struct ArrowArray* array);

/* library / ABI version: major<<16 | minor */
SAILGPU_API uint32_t sailgpu_version(void);

/* Context on CUDA device `device` (ordinal visible to this process). */
SAILGPU_API int32_t sailgpu_ctx_create(int32_t device, sailgpu_ctx** out);
SAILGPU_API void sailgpu_ctx_destroy(sailgpu_ctx* ctx);
/* last error message of a failed ctx-level call (thread-local copy, valid until next call) */
SAILGPU_API const char* sailgpu_ctx_last_error(const sailgpu_ctx* ctx);

/* The CUDA stream (cudaStream_t) every kernel and copy of this context is ordered on, so callers can
 * bracket work with their own CUDA events; and a full synchronisation of that stream. */
SAILGPU_API void* sailgpu_ctx_stream(sailgpu_ctx* ctx);
SAILGPU_API int32_t sailgpu_ctx_synchronize(sailgpu_ctx* ctx);

/* NCCL communicator for the hash-repartition exchange (one rank per GPU/process).
 * unique_id: 128 bytes obtained from sailgpu_comm_unique_id on rank 0 and distributed out of band
 * (the Rust shim sends it in the RunTask message; tests use torch.distributed's store). */
SAILGPU_API int32_t sailgpu_comm_unique_id(uint8_t* out128);
SAILGPU_API int32_t sailgpu_ctx_comm_init(sailgpu_ctx* ctx, const uint8_t* unique_id128, int32_t rank, int32_t world_size);

/* Create an operator.  `input_schemas[i]` is the Arrow schema (struct of fields) of input i;
 * on success *out_schema is filled with the operator's output schema (caller releases it). */
SAILGPU_API int32_t sailgpu_op_create(sailgpu_ctx* ctx, const char* spec_json, size_t spec_len,
                          const struct ArrowSchema* const* input_schemas, int32_t n_inputs,
                          int32_t partition, sailgpu_op** out, struct ArrowSchema* out_schema);

/* Plan-time validation for the rewrite pass (LocalJobRunner::execute, job_runner.rs:63): parses the spec, runs the
 * same type inference as sailgpu_op_create and fills *out_schema, or returns SAILGPU_ERR_UNSUPPORTED / _INVALID with a
 * message in err_buf.  No device is touched, so the decision "GPU node or keep the DataFusion node" is made while
 * planning, never as a silent run-time fallback. */
SAILGPU_API int32_t sailgpu_spec_validate(const char* spec_json, size_t spec_len, const struct ArrowSchema* const* input_schemas,
                                          int32_t n_inputs, struct ArrowSchema* out_schema, char* err_buf, size_t err_cap);

/* Parquet column chunks -> Arrow columns in HBM (the scan before the operator path: DataFusion's DataSourceExec(ParquetSource),
 * crates/sail-data-source/src/listing/planner.rs:47, task_runner/core.rs:115-133).  The caller reads the footer (the Rust side
 * already does, through the `parquet` crate) and hands over, per projected column of ONE row group, the bytes of its column chunk
 * exactly as stored in the file (dictionary page first) plus what the footer says about it; the chunk crosses PCIe as stored and is
 * decoded on the device (page headers and RLE run headers are walked on the host, every value is produced by a GPU thread).
 * `schema` names the Arrow type each column decodes to (Int32/Date32, Int64, Float64, Decimal128 from FIXED_LEN_BYTE_ARRAY /
 * INT32 / INT64, Utf8View from BYTE_ARRAY, Timestamp from INT64 annotated TIMESTAMP(MILLIS|MICROS|NANOS, isAdjustedToUTC): the
 * annotation never reaches the library, the caller names the unit and zone and the 8-byte values pass through unchanged; INT96
 * stays refused).  INT32 also decodes to Int8, Int16, UInt8 and UInt16 (the INT(8|16, signed|unsigned)
 * annotations): the value stored is the low bytes of the INT32, the truncation parquet-cpp and arrow-rs apply.  The library never
 * sees a BYTE_ARRAY column's annotation, so which Arrow type it decodes to is the caller's choice: a UTF8-annotated column and a
 * plain binary one both decode to Utf8View, bytes passed through unchanged and not validated as UTF-8.  A shim applying
 * `binary_as_string` asks for Utf8View for the binary columns.  Covered: data pages V1/V2, PLAIN and dictionary encodings,
 * DELTA_BINARY_PACKED (INT32 / INT64), DELTA_LENGTH_BYTE_ARRAY (BYTE_ARRAY), DELTA_BYTE_ARRAY (BYTE_ARRAY / FIXED_LEN_BYTE_ARRAY)
 * and BYTE_STREAM_SPLIT (DOUBLE / INT32 / INT64 / FIXED_LEN_BYTE_ARRAY), mixed freely within a chunk; a corrupt DELTA stream returns
 * SAILGPU_ERR_INVALID, naming the column (and the page, where the host walk finds it); flat optional columns,
 * uncompressed and ZSTD-compressed pages (codec 0 or 6; columns of both kinds may be mixed in one call); anything else, and
 * ZSTD frames that need a dictionary, returns SAILGPU_ERR_UNSUPPORTED and the caller keeps its CPU reader for that file.
 * ZSTD pages are decompressed on the device by one launch per call, covering every column; the decompressed chunk is read
 * back to the host once, because the RLE run headers are walked there.  A corrupt ZSTD page returns SAILGPU_ERR_INVALID
 * with a message naming the column and the page. */
typedef struct sailgpu_parquet_column {
  const uint8_t* chunk;      /* host pointer: first byte of the column chunk (its dictionary page, else its first data page) */
  uint64_t chunk_len;        /* total_compressed_size of the chunk */
  int32_t physical_type;     /* parquet::Type: 1 INT32, 2 INT64, 5 DOUBLE, 6 BYTE_ARRAY, 7 FIXED_LEN_BYTE_ARRAY */
  int32_t type_length;       /* FIXED_LEN_BYTE_ARRAY length, else 0 */
  int32_t max_def_level;     /* 0 required, 1 optional */
  int32_t codec;             /* parquet::CompressionCodec: 0 UNCOMPRESSED, 6 ZSTD */
  int64_t num_values;
} sailgpu_parquet_column;
SAILGPU_API int32_t sailgpu_parquet_decode(sailgpu_ctx* ctx, const struct ArrowSchema* schema, const sailgpu_parquet_column* cols,
                                           int32_t n_cols, int64_t n_rows, struct ArrowDeviceArray* out);
/* Plan-time / diagnostic companion: walks the pages and run headers of column `column` on the host only and reports what it
 * found as JSON ({"pages":..,"dense":non-null values,"dict_count":..,...,"body_bytes":..,"body_fnv1a":..,"delta_pages":..,
 * "delta_values":..,"bss_pages":..,"bss_values":..}: data pages in a DELTA_* / BYTE_STREAM_SPLIT encoding and their non-null values); fails exactly where
 * sailgpu_parquet_decode would.  body_bytes / body_fnv1a: length and FNV-1a 64 hash of the page bodies walked, in page order,
 * after decompression (a ZSTD chunk is decompressed on the host by the decoder the device runs). */
SAILGPU_API int32_t sailgpu_parquet_inspect(const struct ArrowSchema* schema, const sailgpu_parquet_column* cols, int32_t n_cols,
                                            int64_t n_rows, int32_t column, char* buf, size_t cap);
/* What the last sailgpu_parquet_decode call on `ctx` spent on ZSTD pages, as JSON: {"zstd_pages":..,"zstd_out_bytes":..,
 * "image_bytes":..,"decompress_ms":..,"readback_ms":..} (device time of the decompression launch and of the image read-back,
 * from CUDA events; all zero when the call had no ZSTD column). */
SAILGPU_API int32_t sailgpu_parquet_stats(sailgpu_ctx* ctx, char* buf, size_t cap);

/* Plan-time kernel specialisation.  The library interprets any pipeline at once and, for pipelines that see enough
 * rows (SAILGPU_JIT_MIN_ROWS, default 4 Mi), compiles a specialised sm_90a kernel with NVRTC the first time; the
 * cubin is cached next to the library (or in $SAILGPU_JIT_CACHE).  This call moves that compilation to planning time
 * (the rewrite pass knows the pipelines of a query before the first batch): it generates the kernel for `spec` as it
 * would run over batches whose column i carries a validity buffer iff bit i of `validity_mask` is set, and with
 * SAILGPU_JIT_COMPILE stores its cubin in the cache.  No device is touched.  Returns the cubin size (or the source
 * length without SAILGPU_JIT_COMPILE) and copies the generated source into buf; on failure returns -code and copies
 * the message.  DataFusion has no counterpart: its operators are ahead-of-time compiled Rust. */
#define SAILGPU_JIT_COLD_VARIANT 1   /* the high-cardinality variant of an aggregate (global table only) */
#define SAILGPU_JIT_COMPILE 2
SAILGPU_API int64_t sailgpu_jit_precompile(const char* spec_json, size_t spec_len, const struct ArrowSchema* const* input_schemas,
                                           int32_t n_inputs, uint64_t validity_mask, int32_t flags, char* buf, size_t cap);

/* Hand one input batch (struct array, host memory) to the operator.  Takes ownership: the library
 * calls batch->release when it no longer needs the host buffers (after the H2D copy). */
SAILGPU_API int32_t sailgpu_op_push(sailgpu_op* op, int32_t input_idx, struct ArrowArray* batch);
/* Same for a batch whose buffers are already in HBM (zero copy; released when consumed). */
SAILGPU_API int32_t sailgpu_op_push_device(sailgpu_op* op, int32_t input_idx, struct ArrowDeviceArray* batch);
/* End of stream on input `input_idx`. */
SAILGPU_API int32_t sailgpu_op_finish_input(sailgpu_op* op, int32_t input_idx);

/* Next output batch.  *has_more == 0 and out->length == 0 together mean end of stream.  A batch
 * with has_more == 1 and length == 0 is legal (DataFusion permits empty batches).  When the
 * operator needs more input before it can produce output it returns length 0, has_more 1. */
SAILGPU_API int32_t sailgpu_op_pull(sailgpu_op* op, struct ArrowArray* out, int32_t* has_more);
SAILGPU_API int32_t sailgpu_op_pull_device(sailgpu_op* op, struct ArrowDeviceArray* out, int32_t* has_more);
/* The same batch as a HANDLE for the next GpuExec: `out` carries the length and a release callback but NO column arrays
 * (n_children == 0); the batch stays in the library's internal HBM form -- string views are not rewritten into compact Arrow
 * heaps, no stream is waited for -- and only sailgpu_op_push_device / sailgpu_exchange of this library instance can consume
 * it (an operator of another context waits for the producing context's stream when it takes the handle).  This is what a
 * GpuExec whose parent is a GpuExec pulls: the counterpart of DataFusion handing an Arc<RecordBatch> to the next operator. */
SAILGPU_API int32_t sailgpu_op_pull_device_handle(sailgpu_op* op, struct ArrowDeviceArray* out, int32_t* has_more);

/* For "repartition" operators: output batches of partition `part` only. */
SAILGPU_API int32_t sailgpu_op_pull_partition(sailgpu_op* op, int32_t part, struct ArrowDeviceArray* out, int32_t* has_more);

/* Result sink (SURVEY.md section 8 f3).  Sail sends every result batch to the Spark Connect client as one self-contained Arrow
 * IPC stream -- Schema message, one RecordBatch message, end-of-stream marker (`to_arrow_batch`,
 * crates/sail-spark-connect/src/executor.rs:320-330: StreamWriter::try_new + write + finish).  sailgpu_ipc_stream frames a HOST
 * batch that way (batch == NULL: schema and end-of-stream only) into a malloc'ed buffer the caller returns with
 * sailgpu_ipc_free; it touches no device and needs no context.  sailgpu_op_pull_ipc is sailgpu_op_pull followed by that framing:
 * what the root GpuExec of a plan hands to the executor instead of a RecordBatch.  Column types: those of "Types T" above plus
 * Binary / LargeUtf8 / LargeBinary / BinaryView; nested and dictionary columns return SAILGPU_ERR_UNSUPPORTED. */
SAILGPU_API int32_t sailgpu_ipc_stream(const struct ArrowSchema* schema, const struct ArrowArray* batch, uint8_t** data, size_t* len);
SAILGPU_API int32_t sailgpu_op_pull_ipc(sailgpu_op* op, uint8_t** data, size_t* len, int64_t* rows, int32_t* has_more);
SAILGPU_API const char* sailgpu_ipc_last_error(void);   /* message of the last failed sailgpu_ipc_stream on this thread */
SAILGPU_API void sailgpu_ipc_free(uint8_t* data);

/* All-to-all exchange of the n = world_size device batches in `send` (batch p goes to rank p);
 * on return `recv` holds the concatenation of what every rank sent to this rank.  NCCL
 * send/recv groups over NVLink; counts are exchanged first.  world_size 1 degenerates to a move. */
SAILGPU_API int32_t sailgpu_exchange(sailgpu_ctx* ctx, const struct ArrowSchema* schema,
                         struct ArrowDeviceArray* send, int32_t n, struct ArrowDeviceArray* recv);

/* Metrics as a JSON object with DataFusion's metric names (output_rows, elapsed_compute [ns],
 * output_batches, input_rows, build_time, join_time, ...) plus gpu.* extras
 * (gpu.kernel_ns, gpu.h2d_bytes, gpu.d2h_bytes, gpu.kernel_launches).  Returns bytes needed. */
SAILGPU_API int64_t sailgpu_op_metrics(sailgpu_op* op, char* json_buf, size_t cap);

/* UTF-8 message of the last failed call on this handle ("" if none). */
SAILGPU_API const char* sailgpu_last_error(const sailgpu_op* op);

/* Idempotent; legal at any time (== dropping the RecordBatchStream: cancels and frees HBM). */
SAILGPU_API void sailgpu_op_destroy(sailgpu_op* op);

/* Pinned host memory for callers that want zero-staging H2D (the shim's scan adapter). */
SAILGPU_API int32_t sailgpu_host_alloc(sailgpu_ctx* ctx, size_t bytes, void** out);
SAILGPU_API void sailgpu_host_free(sailgpu_ctx* ctx, void* p);

#ifdef __cplusplus
}
#endif
/* Environment (read by the library; all optional, none changes results):
 *   SAILGPU_JIT=0                 interpret every pipeline;  SAILGPU_JIT_MIN_ROWS=n  rows a pipeline must have seen before it is specialised
 *   SAILGPU_JIT_CACHE=dir         where cubins are kept;  SAILGPU_JIT_VERBOSE / _STRICT / _DUMP  diagnostics of the specialiser
 *   SAILGPU_TOPK_MIN_ROWS=n       TopK selection threshold;  SAILGPU_AGG_MIN_CAPACITY=n  first group-table size
 *   SAILGPU_PACK_THREADS=n        packer threads of the host ingest (default: the CPUs the cgroup grants, at most 32)
 *   SAILGPU_H2D_PACK=0 / SAILGPU_PACK_PIECE_ROWS=n / SAILGPU_PACK_NUMA=0   ingest A/B knobs */

#endif /* SAILGPU_H */
