/*
 * blaze_b200.h — C ABI of the H100-native Filter / Project / HashAgg hot path.
 *
 * This is the drop-in boundary posited by BASELINE.json's north_star: the reference
 * (kwai/blaze = Apache Auron @ d1eaef148a58) keeps its Rust host code — plan-serde, JNI bridge,
 * `ExecutionPlan` impls — and each `execute()` body forwards Arrow batches through these entry
 * points instead of running the CPU operator.  INTEGRATION.md shows the Rust shim.
 *
 * Every entry point names the reference interface it replaces (paths relative to
 * the reference's native-engine/):
 *
 *   b200q_op_create         FilterExec::try_new   datafusion-ext-plans/src/filter_exec.rs:51-73
 *                           ProjectExec::try_new  datafusion-ext-plans/src/project_exec.rs:57-81
 *                           AggExec::try_new      datafusion-ext-plans/src/agg_exec.rs:67-98
 *                           + plan decoding       auron-serde/src/from_proto.rs:107-152,407-500,839-1026
 *   b200q_op_output_schema  ExecutionPlan::schema()        filter_exec.rs:99-101, project_exec.rs:119-121,
 *                                                          agg_exec.rs:121-123
 *   b200q_op_push           the `input.next()` side of the operator loop
 *                           filter_exec.rs:186-195, project_exec.rs:217-229, agg_exec.rs:240-274;
 *                           batch layout = struct-typed ArrowArray, as FFIReaderExec imports it
 *                           datafusion-ext-plans/src/ffi_reader_exec.rs:163-194
 *   b200q_op_finish         end of the input stream: `tables.output(sender)` agg_exec.rs:275
 *   b200q_op_pull           `sender.send(batch)` / SendableRecordBatchStream::poll_next; batches leave
 *                           as struct-typed ArrowArray exactly like auron/src/rt.rs:229-259
 *   b200q_op_metrics        BaselineMetrics / update_spark_metric_node   auron/src/metrics.rs:22-58
 *   b200q_op_destroy        drop of the operator stream / NativeExecutionRuntime::finalize rt.rs:261-273
 *   b200q_conf              auron-jni-bridge/src/conf.rs:32-61 (keys) with the native fallbacks of
 *                           datafusion-ext-commons/src/lib.rs:74-91 and agg/agg_ctx.rs:174-185
 *   b200q_last_error        DataFusionError::Execution(msg) forwarded through the channel
 *                           datafusion-ext-plans/src/common/execution_context.rs:569-598
 *   b200q_murmur3_partition evaluate_hashes + evaluate_partition_ids
 *                           datafusion-ext-plans/src/shuffle/mod.rs:163-188 (Spark murmur3 seed 42, pmod)
 *   ShuffleWriterExecNode plans (b200q_op_create .. b200q_op_finish write <data_file> and <index_file>)
 *                           ShuffleWriterExec::execute        datafusion-ext-plans/src/shuffle_writer_exec.rs:109-165
 *                           SortShuffleRepartitioner          datafusion-ext-plans/src/shuffle/sort_repartitioner.rs:121-185
 *                           BufferedData::write               datafusion-ext-plans/src/shuffle/buffered_data.rs:123-158
 *                           write_batch (byte planes)         datafusion-ext-commons/src/io/batch_serde.rs:66-77,264-306
 *                           IpcCompressionWriter              datafusion-ext-plans/src/common/ipc_compression.rs:34-112
 *   ParquetScanExecNode leaf ParquetExec::execute (decode + row-group pruning)      datafusion-ext-plans/src/parquet_exec.rs:150-203,316-396
 *   SortExecNode plans      SortExec::new + ExternalSorter::insert_batch / output   datafusion-ext-plans/src/sort_exec.rs:97-112,626-752
 *   b200q_op_attach_build   collect_join_hash_map + execute_join_with_map   datafusion-ext-plans/src/broadcast_join_exec.rs:317-385,562-639
 *   b200q_op_attach_right   SortMergeJoinExec::execute (the right child's stream)   datafusion-ext-plans/src/sort_merge_join_exec.rs:200-330
 *   b200q_op_push_ipc       IpcReaderExec::execute (decode of the shuffle blocks)  datafusion-ext-plans/src/ipc_reader_exec.rs:164-272
 *   b200q_op_shuffle_chunk  the per-partition encoded bytes before compression — what BufferedData::write_rss
 *                           hands to an RSS partition writer (buffered_data.rs:160-196)
 *
 * Conventions: every call returns a status (0 = ok) and never unwinds; the message of the last
 * failure on the calling thread is available from b200q_last_error().  A CUDA error is sticky
 * for the handle.  A handle is used by one thread at a time (the operator's producer task);
 * different handles are independent (one CUDA stream set each).
 */
#ifndef BLAZE_B200_H
#define BLAZE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Arrow C Data / Device Data Interface (spec structs; guarded like arrow/c/abi.h) ---------- */
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
#endif /* ARROW_C_DATA_INTERFACE */

#ifndef ARROW_C_DEVICE_DATA_INTERFACE
#define ARROW_C_DEVICE_DATA_INTERFACE
typedef int32_t ArrowDeviceType;
#define ARROW_DEVICE_CPU 1
#define ARROW_DEVICE_CUDA 2
#define ARROW_DEVICE_CUDA_HOST 3

struct ArrowDeviceArray {
  struct ArrowArray array;
  int64_t device_id;
  ArrowDeviceType device_type;
  void* sync_event; /* cudaEvent_t* or NULL */
  int64_t reserved[3];
};
#endif /* ARROW_C_DEVICE_DATA_INTERFACE */

/* ---- status codes ---------------------------------------------------------------------------- */
typedef int32_t b200q_status;
#define B200Q_OK 0
#define B200Q_ERR_INVALID_PLAN 1 /* malformed protobuf / missing required field (PlanSerDeError)   */
#define B200Q_ERR_UNSUPPORTED 2  /* plan is valid for the reference but outside this hot path      */
#define B200Q_ERR_CUDA 3         /* CUDA runtime failure; sticky for the handle                    */
#define B200Q_ERR_STATE 4        /* call sequence violation (push after finish, ...)               */
#define B200Q_ERR_EXECUTION 5    /* data-dependent error, e.g. "Divide by zero error"              */
#define B200Q_ERR_NO_DEVICE 6    /* no CUDA device / sm_90a kernels cannot run: NEVER falls back    */
#define B200Q_ERR_INVALID_ARG 7

/* plan_kind for b200q_op_create / b200q_plan_explain */
#define B200Q_PLAN_NODE 0       /* bytes are a plan.protobuf.PhysicalPlanNode (auron.proto:27-55)  */
#define B200Q_TASK_DEFINITION 1 /* bytes are a plan.protobuf.TaskDefinition   (auron.proto:735-740) */

typedef struct b200q_op b200q_op;

/* Tunables: the AuronConf keys the path reads (AuronConf.java:25-128) + GPU-side sizing knobs. */
typedef struct b200q_conf {
  uint32_t struct_size;               /* sizeof(b200q_conf), for forward compatibility            */
  int32_t batch_size;                 /* BATCH_SIZE, default 10000 (commons/src/lib.rs:74-77)     */
  int64_t suggested_batch_mem_size;   /* SUGGESTED_BATCH_MEM_SIZE, default 8 MiB (lib.rs:79-82)   */
  int32_t partial_agg_skipping_enable;/* accepted; the GPU table never needs to skip (DESIGN.md)  */
  double partial_agg_skipping_ratio;  /* default 0.999 (agg_ctx.rs:177)                           */
  int64_t partial_agg_skipping_min_rows; /* default 20000 (agg_ctx.rs:178)                        */
  int64_t staging_rows;               /* host batches are staged in pinned memory up to this many
                                         rows before one H2D + one kernel launch (default 1<<20)  */
  int64_t agg_initial_groups;         /* initial hash-table sizing hint in groups (default 1<<19) */
  int64_t max_launch_rows;            /* rows per kernel launch for device-resident pushes
                                         (default 1<<27); a sort-merge join also emits its output
                                         in batches of at most this many rows                     */
  int32_t partial_state_columnar;     /* 1: non-final agg output/input uses typed state columns
                                         (GPU-to-GPU exchange) instead of the reference's Binary
                                         frozen-row column `#9223372036854775807`                 */
  int32_t force_generic_kernels;      /* 1: disable the specialised fast kernels (testing)        */
  int32_t agg_dense_keys;             /* 1 (default): single integer keys spanning a small range
                                         are direct-indexed (no probe); 0: always hash           */
  int32_t agg_hot_key_cache;          /* 1 (default): probe the first batch for key skew and, when a
                                         few keys dominate, combine their updates in a CTA-private
                                         shared-memory cache before the global table (DESIGN.md §3) */
  int64_t agg_max_table_bytes;        /* HBM budget of one aggregate's group table (0 = whatever the
                                         device can allocate).  The GPU table never spills: growing
                                         past the budget, or a failed device allocation, returns
                                         B200Q_ERR_UNSUPPORTED so the host falls back to its CPU
                                         operators (replaces spill / partial skipping,
                                         agg/agg_table.rs:108-120,540-588)                       */
  int32_t shuffle_output_on_device;   /* ShuffleWriterExec plans: 1 = keep the encoded partition bytes in HBM (no files are
                                         written; read them with b200q_op_shuffle_chunk), 0 (default) = bring them to the
                                         host and write <data_file>/<index_file> at finish                          */
} b200q_conf;

typedef struct b200q_metrics {
  uint32_t struct_size;
  int64_t input_rows;
  int64_t input_batches;
  int64_t output_rows;                /* BaselineMetrics::output_rows                             */
  int64_t output_batches;
  int64_t elapsed_compute_ns;         /* device time of this op's kernels (CUDA events)           */
  int64_t gpu_kernel_launches;        /* kernels of THIS library launched by the op               */
  int64_t h2d_bytes;
  int64_t d2h_bytes;
  int64_t num_groups;                 /* agg: groups currently in the table                       */
  int64_t table_capacity_slots;
  int64_t table_grow_count;
  int64_t fast_path_launches;         /* launches that took a specialised kernel                  */
  int64_t hot_kernel_ns;              /* CUDA-event time of the dominant kernel only: the HashAgg
                                         update kernel, or the fused filter/project kernel        */
  int64_t hot_kernel_rows;            /* input rows those launches covered                        */
  int64_t hot_kernel_launches;
} b200q_metrics;

/* library identity; safe without a GPU */
int32_t b200q_version(void);
const char* b200q_build_info(void);
/* message of the last failing call on this thread ("" if none) */
const char* b200q_last_error(void);
/* number of visible CUDA devices (0 without a GPU/driver; never an error) */
int32_t b200q_device_count(void);

/* fill *conf with the defaults listed above */
b200q_status b200q_conf_init(b200q_conf* conf);

/* Decode + validate a plan WITHOUT touching the GPU and render it as text (host-logic tests,
 * debugging).  Writes at most cap bytes incl. NUL; *needed = bytes required. */
b200q_status b200q_plan_explain(const uint8_t* plan, size_t plan_len, int32_t plan_kind,
                                char* buf, size_t cap, size_t* needed);

/* Build the operator pipeline for a plan subtree made of Agg / Projection / Filter nodes over one
 * FFIReader or EmptyPartitions leaf.  `input_schema` may be NULL (the leaf carries its schema);
 * when given it must match the leaf schema.  `device` is the CUDA ordinal. */
b200q_status b200q_op_create(const uint8_t* plan, size_t plan_len, int32_t plan_kind,
                             const struct ArrowSchema* input_schema, const b200q_conf* conf,
                             int32_t device, b200q_op** out);

/* schema of the batches accepted by push (the leaf schema) / produced by pull; caller releases */
b200q_status b200q_op_input_schema(b200q_op* op, struct ArrowSchema* out);
b200q_status b200q_op_output_schema(b200q_op* op, struct ArrowSchema* out);

/* Feed one input batch: a struct-typed ArrowArray in HOST memory whose children are the columns
 * of the input schema.  Ownership moves to the library (it calls batch->release when done, also on
 * failure). */
b200q_status b200q_op_push(b200q_op* op, struct ArrowArray* batch);
/* Same, for columns already resident in HBM (ARROW_DEVICE_CUDA, same device as the op). */
b200q_status b200q_op_push_device(b200q_op* op, struct ArrowDeviceArray* batch);

/* End of input: flush staged rows, run final aggregation / emission. */
b200q_status b200q_op_finish(b200q_op* op);

/* Next output batch (struct-typed ArrowArray in host memory; caller releases).  *has_batch = 0
 * when nothing is available: before finish this means "push more", after finish "exhausted". */
b200q_status b200q_op_pull(b200q_op* op, struct ArrowArray* out, int32_t* has_batch);
/* Same, but buffers stay in HBM (for GPU-to-GPU chaining and the HBM-resident benchmark). */
b200q_status b200q_op_pull_device(b200q_op* op, struct ArrowDeviceArray* out, int32_t* has_batch);

/* block until all device work queued by this op has completed */
b200q_status b200q_op_sync(b200q_op* op);

b200q_status b200q_op_metrics(b200q_op* op, b200q_metrics* out);
void b200q_op_destroy(b200q_op* op);

/* ---- Hash join (HashJoinExecNode / BroadcastJoinExecNode + BroadcastJoinBuildHashMapExecNode) --------------------------
 * Reference: BroadcastJoinExec (datafusion-ext-plans/src/broadcast_join_exec.rs:226-298,496-560), the joiners
 * (joins/bhj/full_join.rs:90-379, joins/bhj/semi_join.rs:100-327) and JoinHashMap (joins/join_hash_map.rs:91-275).
 * The map side is its own op, as it is its own plan node in the reference: create an op from a
 * BroadcastJoinBuildHashMapExecNode{input, keys} plan, push the side's batches, finish it — the table and the side's
 * columns stay in HBM.  Create the join op from the HashJoinExecNode / BroadcastJoinExecNode plan (its map-side child only
 * supplies the schema), attach the finished build op, then push the PROBED side's batches and pull the joined rows.
 * Several probe ops (the tasks of a stage) may attach to one build op — the counterpart of the process-wide map cache keyed by
 * cached_build_hash_map_id (broadcast_join_exec.rs:640-677); the build op must outlive them only until they are destroyed
 * (the table is reference counted).  Inner / Left / Right / Full / LeftSemi / LeftAnti / Existence, either side as the map. */
b200q_status b200q_op_attach_build(b200q_op* probe_op, b200q_op* build_op);

/* ---- sort-merge join: the right side (plans with a SortMergeJoinExecNode) -------------------------------------------------
 * Reference: SortMergeJoinExec (datafusion-ext-plans/src/sort_merge_join_exec.rs, joins/smj).  The op created from the
 * SortMergeJoinExecNode subtree takes its LEFT child as its pushed input (push / push_device / push_ipc; stages below the join,
 * typically a SortExec, run in the same op).  `right_op` is an op built from the node's RIGHT child subtree (e.g. IpcReader ->
 * SortExec), finished and not yet pulled: its queued device batches become the join's right side by reference, without a copy
 * when there is one batch (several are concatenated once).  Afterwards b200q_op_pull / pull_device on `right_op` is
 * B200Q_ERR_STATE, and `right_op` may be destroyed (the batches are reference counted).  Status: B200Q_ERR_INVALID_ARG when the
 * right op's output schema differs from the node's right schema, or the right rows are not sorted by the join keys under the
 * node's sort_options; B200Q_ERR_STATE when `right_op` is unfinished or already pulled / attached, when the join op already has
 * a right side or input, and for any push or finish on the join op before this call; B200Q_ERR_UNSUPPORTED for 2^31 right rows
 * or more.  Each side must arrive sorted by its keys: the op checks every left batch, across batch boundaries, and refuses it
 * (B200Q_ERR_INVALID_ARG) instead of returning wrong rows.  Inner / Left / LeftSemi / LeftAnti / Existence output follows the left
 * input order (a left row's rows are contiguous, its matches in right order); Right follows the right keys' order; Full is
 * merged the same way; on equal keys, left-driven rows come before right-only rows. */
b200q_status b200q_op_attach_right(b200q_op* join_op, b200q_op* right_op);

/* ---- ParquetScanExec as the source of an op (plans whose leaf is a ParquetScanExecNode) -----------------------------------
 * Reference: ParquetExec::execute (datafusion-ext-plans/src/parquet_exec.rs:150-203) + the FsProvider byte-range reads
 * (:316-396).  Such an op takes no b200q_op_push: b200q_op_finish reads the split's row groups (FileScanExecConf.file_group,
 * projection, limit; row-group pruning from pruning_predicates), decodes them on the GPU and drives the stages above the scan;
 * pull the result as usual.  Files are opened from the local file system unless a reader is registered — the hook for the host's
 * Hadoop FileSystem bridge (JniBridge.getResource(fsResourceId) in the reference): it must fill dst with bytes
 * [offset, offset + length) of `path` and return 0. */
typedef int32_t (*b200q_file_reader_fn)(void* ctx, const char* path, int64_t offset, int64_t length, uint8_t* dst);
b200q_status b200q_set_file_reader(b200q_file_reader_fn fn, void* ctx);   /* process-wide; fn = NULL restores local files */
/* ---- Scalar subqueries: the bloom filter of BloomFilterMightContain -------------------------------------------------------
 * Reference: SparkScalarSubqueryWrapperExpr::evaluate (datafusion-ext-exprs/src/spark_scalar_subquery_wrapper.rs:109-129), which
 * runs the subquery on the JVM through the wrapper's `serialized` bytes.  Spark's runtime bloom filters place such a wrapper as the
 * filter argument of BloomFilterMightContain; the library evaluates nothing on the JVM, so it asks the host once per
 * BloomFilterMightContain at b200q_op_create (b200q_plan_explain never asks).  `fn` gets the wrapper's serialized bytes and
 * returns 0 after calling `put(sink, value, len)` once with the Binary value (the library copies it before `put` returns), or
 * returns 0 without calling `put` when the value is NULL (the filter then matches no row).  Any other return value fails the
 * create with B200Q_ERR_EXECUTION.  Without a resolver such plans are B200Q_ERR_UNSUPPORTED. */
typedef void (*b200q_bytes_sink_fn)(void* sink, const uint8_t* value, size_t len);
typedef int32_t (*b200q_scalar_subquery_fn)(void* ctx, const uint8_t* serialized, size_t len, b200q_bytes_sink_fn put, void* sink);
b200q_status b200q_set_scalar_subquery_resolver(b200q_scalar_subquery_fn fn, void* ctx);   /* process-wide; fn = NULL removes it */

/* Host-only helpers of the scan (no GPU needed; debugging and the CPU test-suite): render a Thrift-encoded FileMetaData footer
 * (columns with their Arrow mapping, row groups, codecs, statistics) as text; raw Snappy decompression of one page body. */
b200q_status b200q_parquet_explain(const uint8_t* footer, size_t n, char* buf, size_t cap, size_t* needed);
b200q_status b200q_snappy_uncompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_len);

/* ---- ShuffleWriterExec result (plans rooted at ShuffleWriterExecNode) ----------------------------------------
 * Every pushed batch becomes one CHUNK: the rows of the batch grouped by output partition
 * (pmod(murmur3(hash exprs, 42), n), shuffle/mod.rs:163-188) and encoded as the reference's `batch_serde`
 * records (batch_serde.rs:66-77; records of at most conf.batch_size rows).  Binary columns (the frozen accumulator rows of a
 * reference-format AggExec(Partial)) are encoded too: a chunk that carries them cuts records at the reference's suggested batch
 * size for its bytes (compute_suggested_batch_size_for_output, lib.rs:93-116).  Bytes [part_off[p], part_off[p+1]) of
 * `data` are partition p's records of that chunk, UNcompressed.  b200q_op_finish frames them into
 * `u32 length ‖ LZ4 frame` blocks and writes the .data / .index files (unless conf.shuffle_output_on_device).
 * Pointers stay valid until b200q_op_destroy. */
typedef struct b200q_shuffle_chunk {
  const uint8_t* data;        /* host memory, or device memory when on_device = 1 */
  int32_t on_device;
  int32_t num_partitions;
  int64_t rows;
  const uint64_t* part_off;   /* host: num_partitions + 1 byte offsets into data */
  const uint64_t* part_rows;  /* host: rows per partition */
} b200q_shuffle_chunk;
b200q_status b200q_op_shuffle_chunk_count(b200q_op* op, int64_t* out_count);
b200q_status b200q_op_shuffle_chunk(b200q_op* op, int64_t index, b200q_shuffle_chunk* out);
/* The library's LZ4 frame encoder (the compression blocks of the shuffle files; host only, no GPU needed):
 * appends one frame holding src[0, n) to dst (capacity cap); *out_len = frame bytes, or the bytes needed when
 * the call fails with B200Q_ERR_INVALID_ARG because cap is too small. */
b200q_status b200q_lz4_frame_compress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_len);
/* The library's LZ4 frame decoder (host only, no GPU needed): decodes the concatenated frame(s) src[0, n) into dst (capacity
 * cap); *out_len = decoded bytes, or the bytes needed when the call fails with B200Q_ERR_INVALID_ARG because cap is too small.
 * Any frame the LZ4 frame format does not allow (bad magic, reserved bits, truncation, a match before the output start, an
 * overrun, a checksum mismatch) is B200Q_ERR_INVALID_ARG with the byte offset in the message. */
b200q_status b200q_lz4_frame_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_len);

/* ---- IpcReaderExec as the source of an op (plans whose leaf is an IpcReaderExecNode) ------------------------------------
 * Reference: IpcReaderExec::execute (datafusion-ext-plans/src/ipc_reader_exec.rs:164-272), IpcCompressionReader
 * (common/ipc_compression.rs:114-183) and read_batch (datafusion-ext-commons/src/io/batch_serde.rs:79-99).  Such an op takes
 * no b200q_op_push / b200q_op_push_device (B200Q_ERR_STATE); each call hands over the bytes of one BlockObject: a
 * concatenation of `u32 LE length ‖ LZ4 frame` blocks, e.g. one map output's byte range of this partition as its .index file
 * gives it.  The records of consecutive pushes are coalesced into device batches of up to conf.staging_rows rows (b200q_op_finish
 * decodes the rest); a record may straddle two blocks of one push but not two pushes.  The library has finished reading `data`
 * when the call returns.  Malformed bytes -> B200Q_ERR_INVALID_ARG (what is wrong, at which byte of the push); nothing of that
 * push is kept and the handle stays usable.  A zstd frame -> B200Q_ERR_UNSUPPORTED.  b200q_op_push_ipc on an op with another
 * leaf -> B200Q_ERR_STATE. */
b200q_status b200q_op_push_ipc(b200q_op* op, const uint8_t* data, size_t len);

/* Spark-compatible partition ids of device-resident key columns:
 * pid[i] = pmod(murmur3_x86_32 chained over the key columns (NULL leaves the hash unchanged), seed 42,
 * num_partitions).  `keys` is a struct-typed device array; out_pids is a device buffer of
 * keys->array.length uint32.  Used for the multi-GPU partial->final exchange. */
b200q_status b200q_murmur3_partition(const struct ArrowSchema* key_schema,
                                     const struct ArrowDeviceArray* keys, int32_t num_partitions,
                                     uint32_t* out_pids_device, void* cuda_stream);

/* ---- multi-GPU repartitioning (replaces the shuffle between the Partial and the Final AggExec) ----------------
 * Reference: shuffle writer partitioning `evaluate_hashes` + `evaluate_partition_ids`
 * (datafusion-ext-plans/src/shuffle/mod.rs:163-188) and the reduce side feeding `AggExec` Final
 * (agg/agg_ctx.rs:276-301).  One process per GPU; rank r owns partition r of `world` partitions, so GPU partitions
 * equal Spark reduce partitions when world = spark.sql.shuffle.partitions.  Transport: NCCL send/recv over NVLink,
 * bound at run time (dlopen libnccl.so.2); the 128-byte id is an ncclUniqueId the host's control plane distributes. */
typedef struct b200q_exchange b200q_exchange;
b200q_status b200q_exchange_unique_id(uint8_t* out128);               /* rank 0 */
b200q_status b200q_exchange_create(const uint8_t* unique_id128, int32_t rank, int32_t world, int32_t device,
                                   b200q_exchange** out);                /* collective: every rank calls it */
/* Collective.  `in`: struct-typed device array of fixed-width columns (e.g. the columnar partial states), its first
 * n_key_cols children are the grouping keys; ownership moves to the library.  `out`: the rows whose
 * pmod(murmur3(keys, seed 42), world) equals this rank, gathered from all ranks; caller releases. */
b200q_status b200q_exchange_shuffle(b200q_exchange* ex, const struct ArrowSchema* schema,
                                    struct ArrowDeviceArray* in, int32_t n_key_cols, struct ArrowDeviceArray* out);
int64_t b200q_exchange_kernel_launches(const b200q_exchange* ex);
void b200q_exchange_destroy(b200q_exchange* ex);

#ifdef __cplusplus
}
#endif
#endif /* BLAZE_B200_H */
