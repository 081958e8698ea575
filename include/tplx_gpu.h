/*
 * tplx_gpu.h — C ABI of libtplx_gpu.so, the H100 executor for Tuplex's normal-case
 * TransformStage row pipeline.
 *
 * What this boundary replaces in the reference (paths relative to /root/reference/tuplex/):
 *   - IBackend::execute(PhysicalStage*)            core/include/ee/IBackend.h:29-46
 *   - LocalBackend::executeTransformStage          core/src/ee/local/LocalBackend.cc:815-1252
 *   - the JIT'd stage function read_block_f + its per-row callbacks
 *                                                  core/include/physical/CodeDefs.h:43-116
 *   - TransformTask (per-partition hot loop)       core/src/physical/TransformTask.cc:382-513,682-722
 * The deliberate departure from the inner ABI: no per-row callbacks cross the boundary;
 * blocks of rows go in, blocks of rows (+ exception records) come out.
 *
 * Conventions: extern "C", plain pointers and sizes, int32 status codes
 * (0 = OK, negative = tplx_status, message via tplx_gpu_last_error()). Row-level errors never
 * fail a call — they become exception records (IExceptionableTask.h:22-36). Buffers passed in
 * are borrowed for the duration of the call unless stated; buffers handed out are caller-owned
 * (caller allocates, library fills). All entry points are thread-safe per handle.
 * There is NO CPU fallback: every compute entry point fails with TPLX_E_NODEVICE when no
 * CUDA device is usable.
 */
#ifndef TPLX_GPU_H
#define TPLX_GPU_H

#include <stdint.h>
#include "tplx_ir.h"

#ifdef __cplusplus
extern "C" {
#endif

enum tplx_status {
    TPLX_OK = 0,
    TPLX_E_NODEVICE = -1,
    TPLX_E_CUDA = -2,
    TPLX_E_BADDESC = -3,
    TPLX_E_BADARG = -4,
    TPLX_E_NOMEM = -5,
    TPLX_E_UNSUPPORTED = -6,
    TPLX_E_OVERFLOW = -7,
};

typedef struct tplx_stage tplx_stage;   /* replaces TransformStage + compiled functor */
typedef struct tplx_block tplx_block;   /* a device-resident column block (input) */
typedef struct tplx_result tplx_result; /* outputs of one block through a stage */

/* One input column of a column block. Fixed-width types: `data` = n_rows 8-byte values.
 * TPLX_T_STR: `data` = concatenated bytes (no terminators), `offsets` = n_rows+1 uint32.
 * Option[T] columns (utils/include/TypeSystem.h; per-row bitmap in the row format, Serializer.cc:1041-1059) carry a validity
 * bitmap: `valid` = (n_rows + 31) / 32 words, bit (r & 31) of word r >> 5 set = row r holds a value; NULL = no row is None. */
typedef struct tplx_column {
    uint8_t type; /* tplx_type */
    uint8_t pad[7];
    const void *data;
    const uint32_t *offsets;
    uint64_t data_bytes;
    const uint32_t *valid;
} tplx_column;

/* Exception record as produced by the device (fixed width); tplx_gpu_result_exception_partition
 * expands it to the reference layout [rowNo, ecCode, opID, size, row bytes]. */
typedef struct tplx_exception_rec {
    int64_t row;    /* input row index inside the submitted block */
    int64_t row_no; /* TransformTask::_outputRowCounter semantics (TransformTask.cc:764,885) */
    int64_t code;   /* tplx_exception_code / ExceptionCodes.h */
    int64_t op_id;  /* reference operator id */
} tplx_exception_rec;

typedef struct tplx_result_info {
    uint64_t n_in_rows;
    uint64_t n_out_rows;
    uint64_t n_exceptions;
    uint64_t out_str_bytes[TPLX_MAX_COLS]; /* per output column; 0 for fixed-width */
    double kernel_ms;    /* CUDA-event time of the stage kernel(s) on the device stream */
    double total_ms;     /* CUDA-event time submit→results ready (incl. H2D when input was on host) */
    uint32_t kernel_launches;
    uint32_t zero_copy_cols; /* run_host: input columns read in place from page-locked host memory (late materialisation) */
    uint64_t h2d_bytes;      /* run_host: bytes of input explicitly copied host->device */
    uint32_t specialised_launches; /* of kernel_launches: kernels the stage specialiser compiled for this stage (csrc/jit.inl);
                                      0 = the interpreting kernels ran */
    uint32_t lane;                 /* execution lane of the GPU that ran the block: 0 = the primary lane, 1 = the second lane a
                                      concurrent caller takes while the primary one is busy; results not made by a stage run
                                      (hash_finish, joins, merges, ...) report 0 */
} tplx_result_info;

/* ---- process / devices ------------------------------------------------------------------ */
/* Select devices (NULL,0 = device 0 only). Mirrors LocalBackend's executor start-up
 * (LocalEngine.cc:41-115). */
int32_t tplx_gpu_init(const int32_t *devices, int32_t n);
int32_t tplx_gpu_device_count(void);
int32_t tplx_gpu_shutdown(void);
const char *tplx_gpu_last_error(void);
/* name + SM count + memory of a selected device; buf may be NULL */
int32_t tplx_gpu_device_info(int32_t device, char *name_buf, int32_t buf_len, int32_t *sm_count,
                             uint64_t *mem_bytes);

/* ---- stage ------------------------------------------------------------------------------ */
/* desc = serialized tplx_stage_header + sections (tplx_ir.h). Replaces TransformStage::compile
 * (TransformStage.cc:763-914): validates the program and sizes launch configuration. */
int32_t tplx_gpu_stage_create(const void *desc, uint64_t desc_bytes, tplx_stage **out);
int32_t tplx_gpu_stage_destroy(tplx_stage *stage);
/* The stage specialiser (csrc/jit.inl) — this library's counterpart of the reference's per-stage code generation + JIT
 * (StageBuilder.cc:602-1143, TransformStage::compile TransformStage.cc:763-914): for a stage that sees large blocks the op program
 * is printed as a straight-line CUDA row function and the library's own kernel source is compiled around it at run time (NVRTC,
 * sm_90a) and launched instead of the interpreting kernel — same parameters, same tiles / scans / exception records.
 * Controlled by TPLX_JIT (0 off, 1 = stages with blocks of >= TPLX_JIT_MIN_ROWS rows [default], 2 = always); when NVRTC is not
 * installed the interpreting kernels run. This entry point is the diagnostic view of it and needs no device: the generated row
 * function of `kind` (1 = K1 rows, 2 / 3 = K1v with 8 / 4 rows per thread, 4 = K3 aggregate, 5 = K1m mask, 6 = K1w and 10 = K1r,
 * the wide-tile fixed-width kernels; any other number is TPLX_E_BADARG) as text,
 * and, with compile != 0, the size of the cubin NVRTC produced for it (0 + the compiler log when it failed / NVRTC is absent). */
int32_t tplx_gpu_stage_specialise(tplx_stage *stage, int32_t kind, int32_t compile, char *src, uint64_t src_cap, uint64_t *src_len,
                                  uint64_t *cubin_bytes, char *log, uint64_t log_cap);
/* Diagnostic (needs no device): the micro-op program the fixed-width row kernel (K1v) would run for this stage — the planner's
 * accumulator chains, fused compare/filter and dense slot numbers — so that the plan can be checked against the op program on
 * the host. n_uops = 0: the stage is not eligible for K1v. out may be NULL (sizes only); out_slots gets the dense slot of every
 * output column (cap_out entries at most). The reference has no counterpart (LLVM does this inside the JIT, LLVMOptimizer.cc). */
typedef struct tplx_vec_uop {
    uint32_t vop;    /* micro-op (tuplex_b200/csrc/vecvm.cuh: VOp) */
    uint32_t xflags; /* planner flags (VFlag): 1 a<-acc, 2 b<-acc, 4 result not stored, 8 filters, 16 a masked by imm2 */
    uint8_t flags;   /* tplx_instr.flags (constant-operand bits) */
    uint8_t pad0;
    uint16_t opidx;
    uint16_t dst, a, b, c, guard; /* dense slots, TPLX_NOSLOT = none / not in the register file */
    uint16_t pad1;
    int64_t imm, imm2;
} tplx_vec_uop;
int32_t tplx_gpu_stage_vec_plan(const tplx_stage *stage, tplx_vec_uop *out, uint32_t cap, uint32_t *n_uops, uint32_t *n_slots,
                                uint16_t *out_slots, uint32_t cap_out);

/* ---- input blocks ----------------------------------------------------------------------- */
/* Upload a host column block to `device` (pinned or pageable host memory). */
int32_t tplx_gpu_block_upload(int32_t device, const tplx_column *cols, uint32_t n_cols, uint64_t n_rows,
                              tplx_block **out);
/* Wrap columns that already live in device memory on `device` (no copy, caller keeps ownership). */
int32_t tplx_gpu_block_wrap_device(int32_t device, const tplx_column *cols, uint32_t n_cols,
                                   uint64_t n_rows, tplx_block **out);
/* K5: build a column block from reference-format partitions (Partition.h:130-139: int64 numRows then
 * rows in Serializer row format, Serializer.cc:1016-1117) that lie in host memory. */
int32_t tplx_gpu_block_from_partitions(int32_t device, const uint8_t *const *partitions,
                                       const uint64_t *partition_bytes, uint32_t n_partitions,
                                       const uint8_t *col_types, uint32_t n_cols, tplx_block **out);
int32_t tplx_gpu_block_rows(const tplx_block *block, uint64_t *n_rows);
/* Device bytes of every column (values, or string payload + offsets): what a kernel reading the block moves. */
int32_t tplx_gpu_block_column_bytes(const tplx_block *block, uint64_t *bytes, uint32_t max_cols, uint32_t *n_cols);
/* Validity words of an Option[T] column of a block, as stored: (n_rows + 31) / 32 words, tail bits included; `nullable` = 0 for a
 * column without a bitmap (nothing is copied). words may be NULL to ask only for `nullable`. */
int32_t tplx_gpu_block_fetch_validity(const tplx_block *block, uint32_t col, uint32_t *words, uint32_t *nullable);
int32_t tplx_gpu_block_free(tplx_block *block);
/* The rows of n_parts blocks, in order, as one new block on the parts' device that owns its memory (e.g. the build side of a
 * join whose stage produced several block results). Fixed-width columns and string bytes are copied; string offsets are rebased by
 * each part's byte position and validity words realigned to each part's first row, one batched launch per column. A column gets a
 * bitmap when any part has one (a part without one contributes set bits); bits past a part's row count are ignored and the
 * output's tail bits are zero. String buffers are 4-byte-multiple allocations readable up to the next 16-byte boundary. Parts on
 * different devices or with different column counts / types: TPLX_E_BADARG; a string column above 4 GiB: TPLX_E_OVERFLOW. Zero
 * parts give an empty block with no columns on the first initialised device. The parts may be freed when the call returns. */
int32_t tplx_gpu_block_concat(const tplx_block *const *parts, uint32_t n_parts, tplx_block **out);
/* Rows [first_row, first_row + n_rows) of `block`: one piece of tplx_gpu_block_concat_pieces. */
typedef struct tplx_concat_piece {
    const tplx_block *block;
    uint64_t first_row;
    uint64_t n_rows;
} tplx_concat_piece;
/* Per-column flags of tplx_gpu_block_concat_pieces (0 = the column as tplx_gpu_block_concat makes it). */
enum tplx_concat_flags {
    TPLX_CONCAT_DROP_VALID = 1, /* no bitmap in the output: the caller has counted no None in the pieces' rows */
    TPLX_CONCAT_ALL_NONE = 2,   /* None in every row: the output column is TPLX_T_I64 zeros with every validity bit clear; the
                                   pieces' values are not read */
    TPLX_CONCAT_UTF8 = 4,       /* string column: every string is written as CPython's bytes.decode("utf-8", "replace").encode()
                                   gives it (one U+FFFD per maximal invalid subpart); valid strings keep their bytes */
};
/* tplx_gpu_block_concat over row ranges of blocks: the rows of every piece, in order, as one new block that owns its memory.
 * String offsets are rebased from each piece's first offset and validity words realigned from its first row. `col_flags` holds one
 * tplx_concat_flags value per column, or is NULL (all 0). A piece outside its block, or TPLX_CONCAT_UTF8 on a column that is not a
 * string column: TPLX_E_BADARG. A device allocation that fails: TPLX_E_NOMEM, nothing is kept. Other errors as
 * tplx_gpu_block_concat; a string column above 4 GiB after the replacement is TPLX_E_OVERFLOW. The blocks may be freed when the call
 * returns. This is how DataSet.cache() re-blocks stage results into owned blocks. */
int32_t tplx_gpu_block_concat_pieces(const tplx_concat_piece *pieces, uint32_t n_pieces, const uint8_t *col_flags, tplx_block **out);
/* Column statistics of a block (one launch over all columns): none_rows[c] = rows in [0, n_rows) whose validity bit is clear
 * (bits past n_rows are ignored; 0 for a column without a bitmap); invalid_utf8[c] = strings of a string column that
 * TPLX_CONCAT_UTF8 would change, found by validating only the strings of 1024-row tiles whose bytes are not all ASCII (0 for
 * other columns). Both arrays have one entry per column. */
int32_t tplx_gpu_block_stats(const tplx_block *block, uint64_t *none_rows, uint64_t *invalid_utf8);
/* Copy column `col` of a device-resident block to the host: fixed width -> data (n_rows * 8 bytes); TPLX_T_STR -> data (the
 * column's bytes) and offsets (n_rows + 1). data or offsets may be NULL. The block twin of tplx_gpu_result_fetch_column. */
int32_t tplx_gpu_block_fetch_column(const tplx_block *block, uint32_t col, void *data, uint32_t *offsets);
/* A block over the same device memory as `block` that owns none of it (freeing it frees nothing of `block`); `block` must
 * outlive it. Lets a block that several consumers read (a cached dataset) go where the consumer frees its input block. */
int32_t tplx_gpu_block_view(const tplx_block *block, tplx_block **out);
/* The rows of a device-resident block whose bit is set in `keep_words` (bit r & 31 of word r >> 5, (n_rows + 31) / 32 host words; bits
 * past n_rows are ignored), in order, as one new block that owns its memory: every column, string offsets rebased, validity bitmaps
 * realigned (tail bits zero). Built from the stage kernels' survivor list (mask_count / mask_scan / mask_expand) and the row-selector
 * gathers of join and merge outputs. 2^32 - 1 rows or more: TPLX_E_OVERFLOW. `block` may be freed when the call returns. This is how
 * a CPython UDF between two device segments of a stage drops rows from the device blocks. */
int32_t tplx_gpu_block_select(const tplx_block *block, const uint32_t *keep_words, tplx_block **out);
/* Device addresses of column `col` of a device-resident block, as tplx_gpu_block_wrap_device takes them: values or string bytes,
 * string offsets (NULL for fixed width), validity bitmap (NULL without one) and the column's data_bytes; waits for the block's
 * upload. The block must outlive whatever uses them. */
int32_t tplx_gpu_block_device_column(const tplx_block *block, uint32_t col, const void **data, const uint32_t **offsets,
                                     const uint32_t **valid, uint64_t *data_bytes);

/* ---- execution -------------------------------------------------------------------------- */
/* Run the stage over one block (asynchronously on the device's stream; results are complete
 * when tplx_gpu_result_info returns). first_row_no seeds the exception row counter so that
 * several blocks of one task number their rows like TransformTask does (not reset between
 * input partitions of a task, TransformTask.cc:885). Replaces the functor call at
 * TransformTask.cc:702. */
int32_t tplx_gpu_stage_run(tplx_stage *stage, const tplx_block *block, int64_t first_row_no,
                           tplx_result **out);
/* Convenience for host callers: upload + run + free the device block (timed as one unit). */
int32_t tplx_gpu_stage_run_host(tplx_stage *stage, int32_t device, const tplx_column *cols,
                                uint32_t n_cols, uint64_t n_rows, int64_t first_row_no,
                                tplx_result **out);

int32_t tplx_gpu_result_info(tplx_result *res, tplx_result_info *info); /* synchronises */
/* Copy output column `col` to host: fixed-width -> data (n_out_rows*8 bytes);
 * TPLX_T_STR -> data (out_str_bytes[col]) and offsets (n_out_rows+1 uint32). */
int32_t tplx_gpu_result_fetch_column(tplx_result *res, uint32_t col, void *data, uint32_t *offsets);
/* Device pointers of an output column (valid until tplx_gpu_result_free). */
int32_t tplx_gpu_result_device_column(tplx_result *res, uint32_t col, const void **data,
                                      const uint32_t **offsets);
int32_t tplx_gpu_result_fetch_exceptions(tplx_result *res, tplx_exception_rec *recs /* n_exceptions */);
/* AGGREGATE endpoint: the block's partial aggregate, one 8-byte value per accumulator, already
 * combined with the accumulator's init (per-task intermediate, BlockBasedTaskBuilder.cc:185-224). */
int32_t tplx_gpu_result_fetch_aggregate(tplx_result *res, int64_t *acc_bits /* n_accs */);
/* Output rows in the reference's Partition byte format (int64 numRows + Serializer rows),
 * split into partitions of at most partition_bytes like rowToMemorySink (TransformTask.h:47-92).
 * Call with buf == NULL to get the required size and partition count. */
int32_t tplx_gpu_result_partitions(tplx_result *res, uint64_t partition_bytes, uint8_t *buf,
                                   uint64_t buf_bytes, uint64_t *bytes_needed, uint64_t *part_offsets,
                                   uint32_t max_parts, uint32_t *n_parts);
/* Exception rows in the reference's exception-partition format: int64 numRows, then per record
 * int64 rowNo, ecCode, opID, size, followed by the ORIGINAL input row in normal-case input row
 * format (IExceptionableTask.h:22-36, TuplexSourceTaskBuilder.cc:79,186-193). */
int32_t tplx_gpu_result_exception_partition(tplx_result *res, uint8_t *buf, uint64_t buf_bytes,
                                            uint64_t *bytes_needed);
/* K7, CSV sink: the output rows as CSV text, byte for byte what the reference's CSV row writer emits per row
 * (fast_csvwriter, core/src/physical/PipelineBuilder.cc:1550-1722; quoteForCSV, runtime/src/Runtime.cc:682-738):
 * bool -> true / false, i64 -> decimal, str quoted iff it holds the quote char, the delimiter, '\n' or '\r'. No header
 * (LocalBackend::writeOutput adds it per file). f64 -> 8 fixed decimals, correctly rounded (ryu d2fixed(8) digits); a value of
 * magnitude >= 2^63 makes the call return TPLX_E_UNSUPPORTED (host formatter). Call with buf == NULL for the size.
 * Refuses Option[T] output columns (TPLX_E_UNSUPPORTED); tplx_gpu_result_csv_nulls writes them. */
int32_t tplx_gpu_result_csv(tplx_result *res, uint32_t n_cols /* first n_cols output columns, 0 = all */, uint8_t delimiter,
                            uint8_t quotechar, uint8_t *buf, uint64_t buf_bytes, uint64_t *bytes_needed);
/* K7 with None cells: as tplx_gpu_result_csv, and a None cell of an Option[T] output column is written as `null_value`
 * (NUL-terminated), quoted once like a string cell (fast_csvwriter: null_value = quote(null_value)). A null value longer than
 * 128 bytes once quoted returns TPLX_E_UNSUPPORTED. */
int32_t tplx_gpu_result_csv_nulls(tplx_result *res, uint32_t n_cols, uint8_t delimiter, uint8_t quotechar, const char *null_value,
                                  uint8_t *buf, uint64_t buf_bytes, uint64_t *bytes_needed);
int32_t tplx_gpu_result_free(tplx_result *res);

/* ---- hash endpoint (aggregateByKey / unique) ---------------------------------------------- */
/* The per-stage, per-device hash table accumulates over every tplx_gpu_stage_run of the stage
 * (TransformTask.cc:791-866 per-task tables + LocalBackend.cc:2219-2376 merge, done in one
 * table here). hash_finish materialises it as a result whose output columns are
 * key columns followed by one column per accumulator (TransformStage.cc:473-528,568-608). */
int32_t tplx_gpu_stage_hash_reserve(tplx_stage *stage, int32_t device, uint64_t expected_keys);
int32_t tplx_gpu_stage_hash_finish(tplx_stage *stage, int32_t device, tplx_result **out);
/* Merge packed (key columns, accumulator columns) rows — e.g. received from another GPU over
 * NCCL — into this device's table using the accumulators' combine operation. A key column that is
 * an Option key of the stage may carry a validity bitmap (tplx_column.valid; no bitmap = no None);
 * a bitmap on any other column is rejected. */
int32_t tplx_gpu_stage_hash_merge(tplx_stage *stage, const tplx_block *packed);
/* Like hash_finish but the accumulator columns hold raw partials (initial value not applied): the form
 * that is exchanged between GPUs before the owner of a key range merges and finishes. */
int32_t tplx_gpu_stage_hash_export_raw(tplx_stage *stage, int32_t device, tplx_result **out);
/* Drop the device's table (start a new job on the same stage). */
int32_t tplx_gpu_stage_hash_reset(tplx_stage *stage, int32_t device);

/* ---- hash join (K8): build + probe between two column blocks ----------------------------------- */
/* Replaces the reference's pair of stages around a JoinOperator: the build stage that appends every row of the smaller side
 * to the bucket of its key (writeRowToHashTable, core/src/physical/TransformTask.cc:769-842; HashJoinStage.cc) and the probe
 * inside the row pipeline of the other side (addHashJoinProbe + createInnerJoinBucketLoop / createLeftJoinBucketLoop,
 * core/src/physical/PipelineBuilder.cc:2110-2523). Output rows: probe rows in input order, the matches of one probe row in
 * build-row order (bucket order = insertion order); key types i64 / bool / str; a None key matches None keys (null bucket,
 * test/core/JoinTest.cc:21-133). Column order of the result as in JoinOperator::inferSchema (core/src/logical/JoinOperator.cc:163-184):
 * | left non-key columns | key | right non-key columns |. Map / filter stages on either side are ordinary tplx_stage runs whose
 * result columns are wrapped with tplx_gpu_block_wrap_device; the probe shards over devices like any row stage (the table is
 * built once per device: broadcast join, no exchange). */
typedef struct tplx_join tplx_join;
enum tplx_join_flags {
    TPLX_JOIN_LEFT_OUTER = 1,  /* leftJoin: a probe row without a match is emitted once, build columns None (:2214-2328) */
    TPLX_JOIN_BUILD_FIRST = 2, /* the build side is the LEFT dataset (JoinOperator::buildRight() false): its columns come first */
};
/* Build the table over column key_col of a device-resident block. The block is borrowed until tplx_gpu_join_destroy. */
int32_t tplx_gpu_join_build(const tplx_block *build, uint32_t key_col, tplx_join **out);
int32_t tplx_gpu_join_info(const tplx_join *join, uint64_t *n_rows, uint64_t *n_null_rows, double *build_ms, uint32_t *kernel_launches);
/* Probe with a device-resident block on the same device. The result's columns are fetched with the tplx_gpu_result_* calls;
 * nullable output columns (left join, Option inputs) also carry a validity bitmap. */
int32_t tplx_gpu_join_probe(tplx_join *join, const tplx_block *probe, uint32_t key_col, uint32_t flags, tplx_result **out);
int32_t tplx_gpu_join_destroy(tplx_join *join);
/* Validity of output column `col`: *nullable = 1 and (n_out_rows + 31) / 32 words (bit set = value present) when the column
 * can hold None, else *nullable = 0 and `words` untouched. words may be NULL (query only). */
int32_t tplx_gpu_result_fetch_validity(tplx_result *res, uint32_t col, uint32_t *words, uint32_t *nullable);
int32_t tplx_gpu_result_device_validity(tplx_result *res, uint32_t col, const uint32_t **words);

/* ---- in-order merge of resolved rows (K9) --------------------------------------------------------- */
/* Replaces ResolveTask::executeInOrder (core/src/physical/ResolveTask.cc:878-1258, emitNormalRows :300-375) for rows the resolve path
 * produced in the stage's normal-case OUTPUT schema: every resolved row returns to the slot of the task's output stream its exception
 * record occupied (row_no, TransformTask.cc:764,885); exceptions that stay unresolved leave their slot empty. `res` is the stage result
 * of one block run with `first_row_no`; `resolved` is a device-resident block with the stage's visible output columns (validity bitmaps
 * for Option columns), one row per resolved exception, ordered by `resolved_row_nos` (strictly ascending, each the row_no of one of
 * res's exception records). The merged rows come back as a new result (columns + validity, no exception records) that the
 * partition / CSV writers accept like any stage result. */
int32_t tplx_gpu_result_merge_resolved(tplx_result *res, const tplx_block *resolved, const int64_t *resolved_row_nos, int64_t first_row_no,
                                       tplx_result **out);

/* ---- device key sort (K11) ------------------------------------------------------------------ */
/* The rows of any result (a hash_finish result, a stage result, a join probe, a merge) ordered by its first n_keys visible columns,
 * as a new result that owns its columns: the same visible columns, n_out_rows rows, no exception records; `res` is unchanged. The
 * order is the one the Python host path gives groups of one type per column: None first, i64 as signed integers, bool False before
 * True, str by bytes (a string before any longer string it is a prefix of; for valid UTF-8 this is Python's str order); columns
 * compare lexicographically, the first most significant; rows with equal keys keep their input order (stable). `col_flags` is
 * NULL or holds one value per visible column; the only flag it takes is TPLX_CONCAT_DROP_VALID (the caller has counted no None in
 * that column: the output column gets no bitmap). n_keys of 0 or above TPLX_MAX_KEYS, a key column out of range or another flag:
 * TPLX_E_BADARG; an f64 key column: TPLX_E_UNSUPPORTED; 2^31 rows or more: TPLX_E_OVERFLOW; a failed device allocation:
 * TPLX_E_NOMEM, nothing is kept. kernel_ms and kernel_launches of the output's tplx_result_info cover the sort and the gathers. */
int32_t tplx_gpu_result_sort_by_keys(tplx_result *res, uint32_t n_keys, const uint8_t *col_flags, tplx_result **out);

/* ---- multi-GPU: the one exchange step of the path ------------------------------------------- */
/* One rank per (process, device) over NCCL (NVLink 5 / NVSwitch). Map / filter stages shard over ranks without any
 * communication (one task per partition group, LocalBackend.cc:679-735); only aggregate endpoints exchange data:
 * the combine of per-task partial aggregates (TransformTask.cc:218-299, LocalBackend.cc:917-960) and the merge of the
 * per-task hash tables (LocalBackend::createFinalHashmap, LocalBackend.cc:2219-2376). NCCL is resolved at run time
 * (dlopen): without it these calls return TPLX_E_UNSUPPORTED and nothing else in the library is affected. */
#define TPLX_COMM_ID_BYTES 128
/* rank 0 creates the id (ncclGetUniqueId); the host side hands it to every rank by its own means */
int32_t tplx_gpu_comm_unique_id(uint8_t *id /* TPLX_COMM_ID_BYTES */);
/* join: collective over all ranks (ncclCommInitRank); one communicator per device */
int32_t tplx_gpu_comm_init(int32_t device, int32_t rank, int32_t world, const uint8_t *id);
/* one process driving n devices (ncclCommInitAll): rank = position in `devices` */
int32_t tplx_gpu_comm_init_local(const int32_t *devices, int32_t n);
int32_t tplx_gpu_comm_info(int32_t device, int32_t *rank, int32_t *world);
int32_t tplx_gpu_comm_destroy(int32_t device);
/* AGGREGATE endpoint, collective: every rank passes its partial (n_accs raw 8-byte values, e.g. its blocks' results folded in
 * block order); ncclAllGather + a fold in RANK ORDER on the device; every rank receives the same bits (fixed association:
 * f64 sums are reproducible). Without a communicator (or world == 1) the partial is returned unchanged. */
int32_t tplx_gpu_agg_finish(tplx_stage *stage, int32_t device, const int64_t *local_bits, int64_t *out_bits);
/* HASH endpoint, collective: every key gets an owner rank = hash(key) mod world; each rank splits its table by owner on the
 * device, sizes travel in one ncclAllGather, the packed (key, partial) records in grouped ncclSend / ncclRecv between device
 * buffers (all-to-all), and every rank merges what it owns into a fresh table. Afterwards tplx_gpu_stage_hash_finish on
 * rank r yields exactly the groups rank r owns; the union over ranks is the result. No-op for a single rank. */
int32_t tplx_gpu_stage_hash_exchange(tplx_stage *stage, int32_t device);

/* ---- CSV source (K6) ----------------------------------------------------------------------- */
/* Replaces the reference's host CSV source in front of a TransformStage: CSVReader::read +
 * csvmonkey row/cell splitting (core/src/physical/CSVReader.cc:388-634, core/include/physical/csvmonkey.h:523-672)
 * and the cell decoding at the head of the stage function (decodeCells, codegen/src/FlattenedTuple.cc:1215-1330;
 * fast_atoi64 / fast_atod / fast_atob, utils/src/StringUtils.cc:22-255 behind runtime/src/Runtime.cc:319-385).
 * Output: a column block of the rows that fit the normal case (tplx_gpu_stage_run input) and a list of the rows
 * that do not (cell-count mismatch, null value in a non-Option column, conversion error): those go to the
 * interpreter path as BADPARSE_STRING_INPUT / NULLERROR rows do in the reference (CSVReader.cc:470-520,583-600). */
#define TPLX_CSV_SKIP 0xFF /* col_types entry: column is not read (projection pushdown, willBeSerialized = false) */
/* A col_types entry tplx_type | TPLX_T_OPTION reads an Option[T] column (decodeCells, FlattenedTuple.cc:1259-1300): a cell equal
 * to a null value is None (placeholder 0 / empty string in the block, validity bit clear in tplx_block's bitmap, block row order),
 * the row stays in the normal case; a non-null cell decodes as in a T column. An Option column cannot be lazy
 * (TPLX_E_UNSUPPORTED). */
typedef struct tplx_csv_buffer tplx_csv_buffer; /* CSV bytes resident on a device */
typedef struct tplx_csv_result tplx_csv_result;
typedef struct tplx_csv_desc {
    uint8_t delimiter;      /* ',' */
    uint8_t quotechar;      /* '"' */
    uint8_t skip_header;    /* 1: the first row is a header and is dropped (CSVReader.cc:419-449) */
    uint8_t n_null_values;  /* <= 8, together <= 64 bytes */
    uint32_t n_file_cols;   /* cells every row must have */
    const uint8_t *col_types;       /* [n_file_cols] tplx_type or TPLX_CSV_SKIP; at most TPLX_MAX_COLS are read */
    const char *const *null_values; /* compared with the dequoted cell (compareToNullValues) */
    const uint8_t *col_lazy;        /* optional [n_file_cols]: 1 = string column whose bytes stay in the CSV buffer; the block
                                     * carries cell references and tplx_gpu_stage_run materialises the column only for the rows a
                                     * prefilter stage lets through (late materialisation). The buffer must outlive the block. */
} tplx_csv_desc;
typedef struct tplx_csv_bad_row {
    uint32_t row;        /* index among the data rows (header excluded) */
    uint32_t code;       /* TPLX_EC_BADPARSE_STRING_INPUT or TPLX_EC_NULLERROR */
    uint32_t line_start; /* byte range of the row inside the buffer, newline excluded */
    uint32_t line_end;
} tplx_csv_bad_row;
typedef struct tplx_csv_info {
    uint64_t n_rows;   /* data rows found (header excluded) */
    uint64_t n_normal; /* rows in the block */
    uint64_t n_bad;    /* rows for the interpreter path */
    uint32_t sequential_rows; /* 1: irregular quoting, rows were found by the exact sequential kernel */
    uint32_t kernel_launches;
    double parse_ms;   /* CUDA-event time of the parse on the device stream */
} tplx_csv_info;
/* Copy n_bytes (< 4 GiB - 64 KiB) of CSV text to the device (pinned or pageable host memory). */
int32_t tplx_gpu_csv_upload(int32_t device, const void *bytes, uint64_t n_bytes, tplx_csv_buffer **out);
int32_t tplx_gpu_csv_buffer_free(tplx_csv_buffer *buf);
/* Parse a resident buffer into a column block holding the non-skipped columns in file order. */
int32_t tplx_gpu_csv_parse(tplx_csv_buffer *buf, const tplx_csv_desc *desc, tplx_block **out_block,
                           tplx_csv_result **out_res);
int32_t tplx_gpu_csv_result_info(tplx_csv_result *res, tplx_csv_info *info);
int32_t tplx_gpu_csv_result_fetch_bad_rows(tplx_csv_result *res, tplx_csv_bad_row *rows /* n_bad, ascending row */);
int32_t tplx_gpu_csv_result_fetch_rowmap(tplx_csv_result *res, uint32_t *rowmap /* n_normal: block row -> data row */);
/* ends[0 .. n_rows]: ends[i + 1] = byte position of the newline that ends data row i; ends[i] + 1 = first byte that can
 * belong to data row i (leading newlines are skipped); ends[0] = 0xFFFFFFFF when no row precedes data row 0. Lets the host
 * cut the text of any row (interpreter path for rows whose UDF raised). */
int32_t tplx_gpu_csv_result_fetch_row_ends(tplx_csv_result *res, uint32_t *ends /* n_rows + 1 */);
int32_t tplx_gpu_csv_result_free(tplx_csv_result *res);

/* ---- text source (K10) ---------------------------------------------------------------------- */
/* Replaces the host reader of Context.text (python/tuplex/context.py:367-387) and the reference's TextReader
 * (core/src/physical/TextReader.cc:60-140; null values: FileInputOperator.cc:144-149) in front of a TransformStage: a buffer
 * from tplx_gpu_csv_upload becomes a block of one string column, a line per row. Lines end at '\n' (the buffer's appended
 * newline ends an unterminated last line and nothing else); one trailing '\r' is stripped; a line that is not valid UTF-8 is
 * stored as CPython's bytes.decode("utf-8", "replace") gives it (one U+FFFD per maximal invalid subpart); a line equal to a
 * null value after the strip and the replacement is null. With `option`, a null line is None (empty string, validity bit clear
 * in the block's bitmap); without, it is a bad row (TPLX_EC_NULLERROR) for the interpreter path. The result object is the CSV
 * source's: info, bad rows, rowmap and row ends (ends[i] + 1 .. ends[i + 1] = line i, newline excluded) are fetched with the
 * tplx_gpu_csv_result_* calls. A string column above 4 GiB (up to 3x the input after replacement) returns TPLX_E_OVERFLOW. */
typedef struct tplx_text_desc {
    uint8_t n_null_values;          /* <= 8, together <= 64 bytes (UTF-8) */
    uint8_t option;                 /* 1: null lines are None in an Option[str] column; 0: they are bad rows */
    const char *const *null_values; /* NUL-terminated */
} tplx_text_desc;
int32_t tplx_gpu_text_parse(tplx_csv_buffer *buf, const tplx_text_desc *desc, tplx_block **out_block, tplx_csv_result **out_res);

#ifdef __cplusplus
}
#endif
#endif /* TPLX_GPU_H */
