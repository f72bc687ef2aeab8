/*
 * mzgpu.h — C ABI of the H100-native differential-dataflow operator core.
 *
 * This is the drop-in boundary for Materialize's compute-layer hot path
 * (SURVEY.md §8b).  Every entry point replaces one piece of the Rust trait
 * surface that `mz_compute::render` programs against; the reference interface
 * each one stands in for is cited as file:line under /root/reference.
 *
 * Conventions
 *   - plain C: opaque handles, POD rows, pointers + sizes, int32 status codes.
 *     No exceptions or aborts cross this boundary.
 *   - rows are fixed-width little-endian PODs (R16/R32/R40/RA/ROUT below).
 *   - times are totally ordered u64 (mz_repr::Timestamp, src/repr/src/timestamp.rs:41-45).
 *     A frontier (Antichain<u64>) is one u64; MZGPU_FRONTIER_EMPTY is the empty
 *     antichain ("no more times").
 *   - diffs are i64 with wrapping arithmetic (mz_ore::Overflowing<i64> in
 *     release mode, src/ore/src/overflowing.rs:24-35).
 *   - a `mzgpu_ctx` and everything created from it is confined to the thread
 *     that created it (one ctx per timely worker; the reference's operators
 *     are single-threaded Rc<RefCell<..>>, src/compute/src/typedefs.rs:46).
 *   - row pointers carry a memory-space tag (MZGPU_MEM_HOST / MZGPU_MEM_DEVICE).
 *     INPUT row pointers (either space) are read by a copy or kernel enqueued on
 *     the ctx stream: the caller must leave the rows untouched until the next
 *     call that waits for the device (mzgpu_ctx_sync, or anything returning an
 *     exact count).  Pageable host memory is staged by the driver before the
 *     call returns; PINNED host memory and device memory are read in place.
 *   - variable-size results are written to a library-owned device buffer
 *     (`mzgpu_buf`) that the caller downloads or feeds to the next operator.
 *   - calls are asynchronous on the ctx stream.  Data-dependent row counts
 *     (survivors of a consolidation, matches of a probe) stay in device memory
 *     and flow to the next operator there; the `*_buf` entry points chain
 *     operators without a host round trip.  Anything that returns an exact
 *     count to the caller (mzgpu_buf_len, mzgpu_batch_len, a download, ...)
 *     waits for the device once and resolves every outstanding count.  This is
 *     the cooperative-scheduling contract of the reference in GPU form: an
 *     operator returns promptly (yield budgets, src/compute/src/render/join/
 *     linear_join.rs:145-151) and the worker decides when to look at results.
 */
#ifndef MZGPU_H
#define MZGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------- status */
#define MZGPU_OK 0
#define MZGPU_E_INVALID (-1)     /* bad argument / protocol violation            */
#define MZGPU_E_CUDA (-2)        /* sticky CUDA failure: caller panics the worker */
#define MZGPU_E_CAPACITY (-3)    /* caller buffer too small; *n_out = required    */
#define MZGPU_E_UNSUPPORTED (-4) /* plan shape outside the fixed-width subset     */
#define MZGPU_E_NCCL (-5)        /* sticky NCCL failure                           */
#define MZGPU_E_FRONTIER (-6)    /* batch/spine frontier contract violated        */

#define MZGPU_MEM_HOST 0
#define MZGPU_MEM_DEVICE 1

#define MZGPU_FRONTIER_EMPTY UINT64_MAX

/* ------------------------------------------------------------------ rows */
/* (u64 key, i64 diff): BASELINE config 1, `consolidate` on Vec<(u64,i64)>
 * (src/ore/src/iter.rs:260-268). */
typedef struct mzgpu_r16 {
  uint64_t key;
  int64_t diff;
} mzgpu_r16;

/* ((key, val), time, diff): the update triple of every arrangement
 * (KeyValBatcher input, src/compute/src/typedefs.rs:121-126). */
typedef struct mzgpu_r32 {
  uint64_t key;
  uint64_t val;
  uint64_t time;
  int64_t diff;
} mzgpu_r32;

/* join_core result with the identity closure: (key, val1, val2), time, diff
 * (L: FnMut(Key, Val1, Val2), src/compute/src/render/join/mz_join_core.rs:66). */
typedef struct mzgpu_r40 {
  uint64_t key;
  uint64_t val1;
  uint64_t val2;
  uint64_t time;
  int64_t diff;
} mzgpu_r40;

/* Accumulable-reduce update: key -> ((), time, (Vec<Accum>, Diff))
 * (src/compute/src/render/reduce.rs:1313-1334,1861-1903).  This struct is the
 * one-lane row (mzgpu_reduce_new, or mzgpu_reduce_lanes_new with one lane); an
 * operator with C lanes repeats the six lane words C times (see
 * mzgpu_reduce_lanes_new for the table of widths).
 *   total     = Diff component of the pair
 *   non_nulls = Accum::*.non_nulls
 *   acc       = Accum::*.accum as i128 (lo/hi), wrapping
 *   pos_infs / neg_infs / nans = Accum::Float counters (0 for integer SUM) */
typedef struct mzgpu_racc {
  uint64_t key;
  uint64_t time;
  int64_t total;
  int64_t non_nulls;
  uint64_t acc_lo;
  int64_t acc_hi;
  int64_t pos_infs;
  int64_t neg_infs;
  int64_t nans;
  int64_t _pad; /* keeps the row 16-byte aligned (80 B) */
} mzgpu_racc;

/* Reduce output update: (key, finalized aggregates), time, diff (+1/-1)
 * (finalize_accum, src/compute/src/render/reduce.rs:1671-1835).  This struct is
 * the one-lane row; with C lanes the (count, sum_lo, sum_hi) triple repeats C
 * times and flag bits 2l / 2l+1 belong to lane l.
 *   count  = COUNT(col)            = Int64(non_nulls)
 *   sum_lo/sum_hi = SUM(int64)     = i128 (numeric from i128);
 *                   SUM(f64)       = f64 bits in sum_lo, sum_hi = 0
 *   flags  bit0: SUM is NULL (total>0 && accum.is_zero())
 *          bit1: error row "net-zero records with non-zero accumulation"
 *                (reduce.rs:1418-1429) */
typedef struct mzgpu_rout {
  uint64_t key;
  int64_t count;
  uint64_t sum_lo;
  int64_t sum_hi;
  uint64_t flags;
  uint64_t time;
  int64_t diff;
  int64_t _pad;
} mzgpu_rout;

/* ---------------------------------------------------------- descriptors */
/* Batch description: Description{lower, upper, since}
 * (differential_dataflow::trace::Description; A3 in SURVEY.md). */
typedef struct mzgpu_desc {
  uint64_t lower;
  uint64_t upper;
  uint64_t since;
} mzgpu_desc;

/* Closure descriptor: the fixed-width stand-in for JoinClosure
 * (src/compute-types/src/plan/join.rs:50-82) and for the key/val plans of
 * render_reduce (src/compute-types/src/plan/reduce.rs:517-522).  Columns are
 * bit-fields of the three 64-bit source words (key, stream val, lookup val).
 *   out.key = OR over key_fields of  field(src) << dst_shift
 *   out.val = OR over val_fields of  field(src) << dst_shift
 *             or, if expr_kind == MZGPU_EXPR_MUL_CONST_MINUS,
 *             field(expr_a) * (expr_c - field(expr_b))     (wrapping i64)
 *   the row is dropped unless every filter holds.
 * Anything richer is MZGPU_E_UNSUPPORTED at plan time (the host keeps its own
 * path for such dataflows; there is no CPU fallback inside the core). */
#define MZGPU_SRC_KEY 0
#define MZGPU_SRC_VAL1 1 /* stream row value   */
#define MZGPU_SRC_VAL2 2 /* lookup row value   */

typedef struct mzgpu_field {
  uint8_t src;       /* MZGPU_SRC_*                 */
  uint8_t shift;     /* right shift of source word  */
  uint8_t bits;      /* field width 1..64           */
  uint8_t dst_shift; /* left shift in the out word  */
} mzgpu_field;

#define MZGPU_CMP_EQ 0
#define MZGPU_CMP_NE 1
#define MZGPU_CMP_LT 2
#define MZGPU_CMP_LE 3
#define MZGPU_CMP_GT 4
#define MZGPU_CMP_GE 5

typedef struct mzgpu_filter {
  mzgpu_field field; /* dst_shift unused */
  uint32_t op;       /* MZGPU_CMP_*, unsigned compare */
  uint64_t rhs;
} mzgpu_filter;

#define MZGPU_EXPR_NONE 0
#define MZGPU_EXPR_MUL_CONST_MINUS 1 /* a * (c - b) */

#define MZGPU_MAX_FIELDS 6
#define MZGPU_MAX_FILTERS 4

typedef struct mzgpu_closure {
  uint32_t n_key_fields;
  uint32_t n_val_fields;
  uint32_t n_filters;
  uint32_t expr_kind;
  mzgpu_field key_fields[MZGPU_MAX_FIELDS];
  mzgpu_field val_fields[MZGPU_MAX_FIELDS];
  mzgpu_filter filters[MZGPU_MAX_FILTERS];
  mzgpu_field expr_a;
  mzgpu_field expr_b;
  uint64_t expr_c;
} mzgpu_closure;

/* half_join time comparison: `le` if source relation < lookup relation else
 * `lt` (src/compute/src/render/join/delta_join.rs:204-224). */
#define MZGPU_HALFJOIN_LE 0
#define MZGPU_HALFJOIN_LT 1

/* Aggregate kinds of the reduce operator.  MZGPU_AGG_COUNT_SUM_* accumulate one
 * value column with mzgpu_reduce_new, and are the lane kinds of
 * mzgpu_reduce_lanes_new, which accumulates up to eight columns in one
 * arrangement (AccumulablePlan, src/compute-types/src/plan/reduce.rs:146-158). */
#define MZGPU_AGG_COUNT_SUM_I64 0 /* COUNT(val), SUM(val) with val: int64   */
#define MZGPU_AGG_COUNT_SUM_F64 1 /* COUNT(val), SUM(val) with val: float64 */
/* ReducePlan::Distinct (build_distinct, src/compute/src/render/reduce.rs:264-334): the
 * arrangement key is the whole row (val is ignored); the output holds (key, ()) once while
 * the key's accumulated multiplicity is non-zero.  ROUT rows: count = 1, sums = 0, flags
 * bit1 = "Non-positive multiplicity in DistinctBy" (the DistinctByErrorCheck reduce). */
#define MZGPU_AGG_DISTINCT 2
/* ThresholdPlan::Basic (threshold_arrangement, src/compute/src/render/threshold.rs:33-77):
 * rows with a positive accumulated multiplicity are kept WITH that multiplicity.  The key is
 * the whole row; ROUT rows carry count = sums = flags = 0 and diff = the change of
 * max(multiplicity, 0). */
#define MZGPU_AGG_THRESHOLD 3
/* MIN(val) / MAX(val) per key: the result of the hierarchical reduce
 * (build_bucketed / build_bucketed_negated_output, src/compute/src/render/reduce.rs:796-1135):
 * over the accumulated (value, count) pairs of the key with non-zero count, any non-positive
 * count yields the error row ("Non-positive accumulation in MinsMaxesHierarchical", flags bit1),
 * otherwise func(values).  Values compare as unsigned 64-bit integers.  ROUT rows: sum_lo = the
 * aggregate, count = sum_hi = 0.  The reference buckets large groups into a reduction tree; this
 * operator evaluates a key's values directly, for any number of distinct live values (a key with more
 * than 32 is walked in value order over its runs).  An activation is evaluated in one pass: a sealed
 * batch of more than 24 Mi rows (MIN / MAX) is refused with MZGPU_E_UNSUPPORTED and the operator
 * reports that status from then on.  The limit applies to the batch's actual row count: a sealed batch
 * whose length bound is past it (such as one sealed from a device-resident input whose buffer bound is
 * loose) has its length read back first, and runs if the rows fit. */
#define MZGPU_AGG_MIN 4
#define MZGPU_AGG_MAX 5
/* TopK per key (BasicTopKPlan, src/compute/src/render/top_k.rs:215-248 and the reduction logic of
 * build_topk_negated_stage, :521-673): over the key's live (value, count) pairs -- any non-positive
 * count yields the error row (flags bit1, diff 1); otherwise the values are ordered (ascending, or
 * descending), `offset` rows are skipped and at most `limit` rows kept, counting multiplicities.
 * The operator emits the changes of that window directly (the reference emits its negated complement
 * and concatenates it with the input: the same collection).  ROUT rows: sum_lo = the value,
 * diff = the change of the value's multiplicity inside the window, count = sum_hi = 0.  The staged
 * bucket tree (build_topk, :251-380) bounds per-key work for huge groups; here, as for MIN/MAX, groups
 * of any width are evaluated, and only a WINDOW of more than 32 distinct values (LIMIT above 32, or
 * none, on a key that wide) is reported MZGPU_E_UNSUPPORTED (at the next read-back; the report poisons
 * the context).  The single-pass bound is 48 Mi / (2 * min(limit, 32) + 2) rows of the sealed batch
 * (LIMIT NULL counts as 32: 762,600 rows; LIMIT 1: 12 Mi), refused as for MIN / MAX.  Created by
 * mzgpu_topk_new. */
#define MZGPU_AGG_TOPK 6

/* ---------------------------------------------------------------- handles */
typedef struct mzgpu_ctx mzgpu_ctx;         /* one per timely worker / GPU            */
typedef struct mzgpu_buf mzgpu_buf;         /* library-owned growable device row buffer */
typedef struct mzgpu_batcher mzgpu_batcher; /* MergeBatcher analogue                  */
typedef struct mzgpu_batch mzgpu_batch;     /* Rc<OrdValBatch> analogue (refcounted)  */
typedef struct mzgpu_spine mzgpu_spine;     /* Spine / TraceAgent analogue            */
typedef struct mzgpu_join mzgpu_join;       /* mz_join_core operator state            */
typedef struct mzgpu_reduce mzgpu_reduce;   /* accumulable reduce operator state      */

/* ---------------------------------------------------------------- context */
/* One context per timely worker thread: device ordinal, worker index, peers
 * (TimelyConfig, src/cluster-client/src/client.rs:19-41). */
int32_t mzgpu_ctx_create(int32_t device, int32_t worker_index, int32_t peers, mzgpu_ctx** out);
void mzgpu_ctx_destroy(mzgpu_ctx* ctx);
/* Thread-local message for the last failing call on this ctx (never NULL). */
const char* mzgpu_last_error(mzgpu_ctx* ctx);
/* Block until all queued device work of this ctx is complete. */
int32_t mzgpu_ctx_sync(mzgpu_ctx* ctx);
/* Counters for the metrics the reference exports per arrangement
 * (src/compute/src/extensions/arrange.rs:210-308) plus kernel launch count. */
typedef struct mzgpu_stats {
  uint64_t kernel_launches;
  uint64_t device_bytes_in_use;
  uint64_t device_bytes_peak;
  uint64_t rows_in;
  uint64_t rows_out;
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
  uint64_t host_syncs; /* times the host waited for the device */
} mzgpu_stats;
int32_t mzgpu_ctx_stats(mzgpu_ctx* ctx, mzgpu_stats* out);
/* Host-side time accounting since the ctx was created: out[0] = ns spent WAITING for the device
 * (the host_syncs above), out[1] = ns spent inside the allocator, out[2] = allocations, out[3] =
 * bytes allocated.  The measurement harness uses it to tell host work from host waiting. */
int32_t mzgpu_ctx_host_times(mzgpu_ctx* ctx, uint64_t out[4]);
/* Per-kernel device timing (CUDA events on the ctx stream around every launch).
 * Off by default; the measurement harness switches it on for a profiling pass
 * (it adds two event records per launch).  mzgpu_profile_report writes one line
 * per kernel: "name launches total_ms algorithmic_bytes\n", NUL terminated;
 * returns MZGPU_E_CAPACITY if `cap` is too small.  Reading the report resets it. */
int32_t mzgpu_profile_enable(mzgpu_ctx* ctx, int32_t on);
int32_t mzgpu_profile_report(mzgpu_ctx* ctx, char* buf, uint64_t cap);
/* Phase timing of the fused consolidate kernel's launches since profiling was
 * enabled: 32 words per launch ([0..9] globaltimer ns at the phase boundaries,
 * [16] rows, [17] radix rounds, [18] bits per round (8 bits each), [19] CTAs). */
int32_t mzgpu_profile_fused_phases(mzgpu_ctx* ctx, uint64_t* out, uint32_t cap_records, uint32_t* n);
/* The CUDA stream all of this ctx's work is issued on (a cudaStream_t), so a
 * host harness can bracket it with its own events. */
void* mzgpu_ctx_stream(mzgpu_ctx* ctx);

/* ------------------------------------------------------------ row buffers */
#define MZGPU_ROW_R16 16
#define MZGPU_ROW_R32 32
#define MZGPU_ROW_R40 40
#define MZGPU_ROW_RACC 80
#define MZGPU_ROW_ROUT 64

int32_t mzgpu_buf_new(mzgpu_ctx* ctx, uint32_t row_bytes, mzgpu_buf** out);
void mzgpu_buf_free(mzgpu_buf* buf);
uint64_t mzgpu_buf_len(const mzgpu_buf* buf);
uint32_t mzgpu_buf_row_bytes(const mzgpu_buf* buf);
/* Device pointer to the rows (valid until the next call that writes `buf`). */
void* mzgpu_buf_device_ptr(mzgpu_buf* buf);
/* Replace the contents with `n` rows from host or device memory. */
int32_t mzgpu_buf_upload(mzgpu_buf* buf, const void* rows, uint64_t n, int32_t mem);
/* Append `n` rows. */
int32_t mzgpu_buf_append(mzgpu_buf* buf, const void* rows, uint64_t n, int32_t mem);
/* Copy rows out; MZGPU_E_CAPACITY (with *n_out = len) if cap is too small. */
int32_t mzgpu_buf_download(mzgpu_buf* buf, void* rows, uint64_t cap, int32_t mem, uint64_t* n_out);
int32_t mzgpu_buf_clear(mzgpu_buf* buf);
/* Append the rows of `src` (same row width) without reading its length back. */
int32_t mzgpu_buf_append_buf(mzgpu_buf* dst, mzgpu_buf* src);
/* The same where the caller knows a tighter bound on src's row count than the library does
 * (`dst` then grows by at most `max_rows`, not by src's internal upper bound): e.g. collecting a
 * reduce's few output corrections timestamp after timestamp.  More rows than `max_rows` are
 * detected on the device: MZGPU_E_CAPACITY at the next read-back, nothing out of bounds. */
int32_t mzgpu_buf_append_buf_at_most(mzgpu_buf* dst, mzgpu_buf* src, uint64_t max_rows);

/* ---------------------------------------------------- a1: consolidation */
/* differential_dataflow::consolidation::consolidate on Vec<(u64,i64)>:
 * sort by key, sum diffs of equal keys, drop zeros (callers e.g.
 * src/compute/src/render/join/delta_join.rs:649; pinned by
 * src/ore/src/iter.rs:260-268).  In place; *n_out = surviving rows. */
int32_t mzgpu_consolidate_r16(mzgpu_ctx* ctx, mzgpu_r16* rows, uint64_t n, int32_t mem,
                              uint64_t* n_out);
/* consolidate_updates on Vec<((K,V),T,R)>: sort by (key,val,time), sum, drop
 * zeros (src/compute/src/render/join/mz_join_core.rs:563; reference model
 * src/timely-util/src/columnar/batcher.rs:1116-1130). */
int32_t mzgpu_consolidate_r32(mzgpu_ctx* ctx, mzgpu_r32* rows, uint64_t n, int32_t mem,
                              uint64_t* n_out);
/* Same on a device buffer (R16 / R32 / R40 / RACC by row_bytes), in place. */
int32_t mzgpu_buf_consolidate(mzgpu_buf* buf);

/* ------------------------------------------ a2-a5: batcher and batches */
/* Batcher::new (src/timely-util/src/operator.rs:572-575).  row_bytes selects
 * R32 (KeyValBatcher) or RACC (the accumulable arrangement's batcher).  R40 rows
 * (the hierarchical MIN / MAX reduce's arrangement) are accepted as well, by
 * batchers, builders and spines alike. */
int32_t mzgpu_batcher_new(mzgpu_ctx* ctx, uint32_t row_bytes, mzgpu_batcher** out);
void mzgpu_batcher_free(mzgpu_batcher* b);
/* Batcher::push_container: sort + consolidate the container into a chain and
 * keep chains geometric (Chunker::push_into,
 * src/timely-util/src/columnar/batcher.rs:65-122; Merger::merge :635-753). */
int32_t mzgpu_batcher_push(mzgpu_batcher* b, const void* rows, uint64_t n, int32_t mem);
/* push_container for rows that already sit in a device buffer (no length read-back). */
int32_t mzgpu_batcher_push_buf(mzgpu_batcher* b, mzgpu_buf* rows);
/* Batcher::seal::<Builder>(upper): merge all chains, ship updates with
 * !upper.less_equal(time), keep the rest (InternalMerge::extract,
 * src/timely-util/src/columnation.rs:636-655), build the batch with
 * Description{lower = previous upper, upper, since = 0}.  *new_lower is the
 * batcher frontier afterwards (min kept time or MZGPU_FRONTIER_EMPTY). */
int32_t mzgpu_batcher_seal(mzgpu_batcher* b, uint64_t upper, mzgpu_batch** batch_out,
                           uint64_t* new_lower);
/* Seal k distinct batchers of one context at the same frontier: the k arrangements a timely
 * worker seals when a timestamp closes (one `Batcher::seal` per arrange operator,
 * src/compute/src/extensions/arrange.rs:86-119, all activated by the same frontier advance).
 * Results are those of k mzgpu_batcher_seal calls in this order; the update-batch-sized seals
 * share one cooperative launch, so k seals cost about one. */
int32_t mzgpu_batcher_seal_many(uint32_t k, mzgpu_batcher* const* batchers, uint64_t upper,
                                mzgpu_batch** batches_out);
/* Batcher::frontier (operator.rs:618-631). */
uint64_t mzgpu_batcher_frontier(const mzgpu_batcher* b);
/* Updates currently buffered. */
uint64_t mzgpu_batcher_len(const mzgpu_batcher* b);

/* Build a batch directly from unsorted updates with an explicit description
 * (Builder::seal, operator.rs:647-677): sort + consolidate + index. */
int32_t mzgpu_batch_build(mzgpu_ctx* ctx, uint32_t row_bytes, const void* rows, uint64_t n,
                          int32_t mem, mzgpu_desc desc, mzgpu_batch** out);
uint64_t mzgpu_batch_len(const mzgpu_batch* b);  /* Batch::len = #updates */
uint64_t mzgpu_batch_keys(const mzgpu_batch* b); /* distinct keys         */
mzgpu_desc mzgpu_batch_desc(const mzgpu_batch* b);
void mzgpu_batch_retain(mzgpu_batch* b);  /* Rc::clone */
void mzgpu_batch_release(mzgpu_batch* b); /* drop      */
/* Cursor walk of the whole batch in (key,val,time) order into caller memory. */
int32_t mzgpu_batch_export(mzgpu_batch* b, void* rows, uint64_t cap, int32_t mem,
                           uint64_t* n_out);
/* ---- a8: cursors over a batch (BatchReader::cursor; the walk mz_join_core does at
 * src/compute/src/render/join/mz_join_core.rs:606-621,816-837 and walk_cursor at
 * src/compute/src/render/context.rs:1299-1355), in batched form: a round trip to the
 * device per seek_key would waste the machine, so a seek takes N keys and a scan takes
 * a page of keys.  A host-side Cursor (rust-shim/src/cursor.rs) keeps the returned
 * runs and rows and answers get_key / step_key / get_val / step_val / map_times from
 * them: rows of a run are in (val, time) order, so step_val is "next row whose val
 * differs" and map_times is "the rows that share the val". */
typedef struct mzgpu_key_run {
  uint64_t key;   /* Cursor::key after the seek (valid iff len != 0)            */
  uint64_t first; /* index of the key's first update row in the batch           */
  uint64_t len;   /* update rows of that key; 0 = key_valid() is false (the end) */
} mzgpu_key_run;
/* Cursor::seek_key for n keys at once: runs[i] describes the first key >= keys[i]
 * (seek_key's position; exact match iff runs[i].key == keys[i]).  keys / runs live
 * in `mem` space. */
int32_t mzgpu_batch_seek_keys(mzgpu_batch* b, const uint64_t* keys, uint64_t n, int32_t mem,
                              mzgpu_key_run* runs);
/* Cursor::rewind_keys + step_key in pages: the distinct keys with ordinals
 * [first_ordinal, first_ordinal + max_keys) in key order, with their runs.
 * *n_out = keys written (fewer than max_keys at the end of the batch). */
int32_t mzgpu_batch_key_page(mzgpu_batch* b, uint64_t first_ordinal, uint64_t max_keys, int32_t mem,
                             mzgpu_key_run* runs, uint64_t* n_out);
/* The update rows [first, first + len) of the batch in cursor order -- get_val /
 * step_val / map_times over one or several consecutive key runs -- into caller memory
 * (rows of the batch's row width). */
int32_t mzgpu_batch_rows(mzgpu_batch* b, uint64_t first, uint64_t len, void* rows, int32_t mem);
/* The batch's hash index, for tests and diagnostics (read-only): *n_slots table slots of 16
 * bytes {key, meta} into `slots` (in `mem` space; MZGPU_E_CAPACITY with the three counts set if
 * cap_slots < *n_slots), the distinct keys, and the longest key run (saturating at 1024).  A slot
 * with meta == 0 is empty; otherwise meta bits [0, 44) hold the key's first row + 1 and bits
 * [44, 64) its run length, or 0 where the builder left the run to the reader. */
int32_t mzgpu_batch_index_export(mzgpu_batch* b, void* slots, uint64_t cap_slots, int32_t mem, uint64_t* n_slots,
                                 uint64_t* n_keys, uint64_t* longest_run);

/* ---- a5: Builder::{with_capacity, push, done} (src/timely-util/src/operator.rs:634-677;
 * OrdValBuilder): chunks of updates are pushed in order, `done` seals them into a batch
 * with the given description.  The builder accepts any chunk order (it sorts and
 * consolidates at `done`, which is a no-op on the sorted, consolidated chains a Batcher
 * hands over), so it also serves as "arrange this collection". */
typedef struct mzgpu_builder mzgpu_builder;
int32_t mzgpu_builder_new(mzgpu_ctx* ctx, uint32_t row_bytes, uint64_t capacity_rows, mzgpu_builder** out);
void mzgpu_builder_free(mzgpu_builder* b);
int32_t mzgpu_builder_push(mzgpu_builder* b, const void* rows, uint64_t n, int32_t mem);
int32_t mzgpu_builder_push_buf(mzgpu_builder* b, mzgpu_buf* rows);
/* Consumes the pushed rows; the builder is empty afterwards and can be reused. */
int32_t mzgpu_builder_done(mzgpu_builder* b, mzgpu_desc desc, mzgpu_batch** out);

/* Batch::Merger::{begin_merge,work,done} in one call (a7): merge two adjacent
 * batches (b1.upper == b2.lower), advance times by `since`, consolidate. */
int32_t mzgpu_batch_merge(mzgpu_batch* b1, mzgpu_batch* b2, uint64_t since, mzgpu_batch** out);

/* --------------------------------------------- a6, a8, a14: the spine */
/* Spine::new with the fuel multiplier `effort` (spine_fueled; in-tree fork
 * src/persist-client/src/internal/trace.rs:1668-1691). */
int32_t mzgpu_spine_new(mzgpu_ctx* ctx, uint32_t row_bytes, uint32_t effort, mzgpu_spine** out);
void mzgpu_spine_free(mzgpu_spine* s);
/* Trace::insert (trace.rs:1737-1770). Takes a reference on `batch`. */
int32_t mzgpu_spine_insert(mzgpu_spine* s, mzgpu_batch* batch);
/* Trace::exert (trace.rs:1698-1727); *did_work mirrors its bool result. */
int32_t mzgpu_spine_exert(mzgpu_spine* s, uint64_t effort, int32_t* did_work);
/* Materialize's ExertionLogic (src/cluster/src/client.rs:227-254): returns the
 * effort to exert now (1000) or 0. */
uint64_t mzgpu_spine_exert_logic(const mzgpu_spine* s, uint32_t proportionality);
/* TraceReader::{set,get}_{logical,physical}_compaction
 * (src/compute/src/arrangement/manager.rs:174-219). */
int32_t mzgpu_spine_set_logical_compaction(mzgpu_spine* s, uint64_t frontier);
int32_t mzgpu_spine_set_physical_compaction(mzgpu_spine* s, uint64_t frontier);
uint64_t mzgpu_spine_get_logical_compaction(const mzgpu_spine* s);
uint64_t mzgpu_spine_get_physical_compaction(const mzgpu_spine* s);
/* TraceReader::read_upper (mz_join_core.rs:337). */
uint64_t mzgpu_spine_read_upper(const mzgpu_spine* s);
/* cursor_through(upper): the batches whose upper <= `upper`, oldest first
 * (mz_join_core.rs:243-246).  Borrowed pointers, valid until the next call
 * that mutates the spine.  MZGPU_E_CAPACITY if cap is too small. */
int32_t mzgpu_spine_batches_through(mzgpu_spine* s, uint64_t upper, mzgpu_batch** batches,
                                    uint32_t cap, uint32_t* n_out);
/* Layer structure for tests against the reference's datadriven traces
 * (src/persist-client/tests/trace/compaction): for each layer, largest first,
 * writes {n_batches, len(b0), len(b1), merge_remaining_work}. */
int32_t mzgpu_spine_layers(const mzgpu_spine* s, uint64_t* out4, uint32_t cap_layers,
                           uint32_t* n_layers);
/* ArrangementSize (src/compute/src/extensions/arrange.rs:210-308 logs size, capacity and
 * allocations of every arrangement through its batches' heap_size): the same three
 * numbers for this spine's batches (admitted and pending).  size = bytes of live update
 * rows and occupied index slots, capacity = bytes of the device allocations backing
 * them, allocations = number of device allocations.  Never waits for the device: a
 * batch whose length is still in flight counts with its upper bound. */
typedef struct mzgpu_arrangement_size {
  uint64_t size_bytes;
  uint64_t capacity_bytes;
  uint64_t allocations;
  uint64_t batches;
  uint64_t updates; /* sum of batch lengths (upper bound while in flight) */
} mzgpu_arrangement_size;
int32_t mzgpu_spine_size(const mzgpu_spine* s, mzgpu_arrangement_size* out);
/* as_collection / walk_cursor (src/compute/src/render/context.rs:1299-1355):
 * the consolidated contents of the whole trace, times advanced to `since`. */
int32_t mzgpu_spine_export(mzgpu_spine* s, mzgpu_buf* out);

/* ------------------------------------------------------ a9: join_core */
/* mz_join_core over two arrangements (mz_join_core.rs:56-455).  `closure`
 * NULL = identity: results are R40 (key,val1,val2); otherwise R32. */
int32_t mzgpu_join_new(mzgpu_ctx* ctx, mzgpu_spine* trace1, mzgpu_spine* trace2,
                       const mzgpu_closure* closure, mzgpu_join** out);
void mzgpu_join_free(mzgpu_join* j);
/* A new batch arrived on input `side` (0 or 1) with capability time `cap`:
 * enqueue (batch x cursor_through(other, ack_other)) and advance ack_side
 * (mz_join_core.rs:218-327). */
int32_t mzgpu_join_core_push(mzgpu_join* j, int32_t side, mzgpu_batch* batch, uint64_t cap);
/* Work::process (mz_join_core.rs:534-582): run deferred work until `fuel_rows`
 * results were produced; results (consolidated per work item) are appended to
 * `out`; *done = 1 when the queue is empty. */
int32_t mzgpu_join_core_work(mzgpu_join* j, uint64_t fuel_rows, mzgpu_buf* out, int32_t* done);
/* The same with the reference's yield function (YieldSpec,
 * src/compute/src/render/join/linear_join.rs:145-151: stop after `fuel_rows` of work OR
 * after a time budget): work stops at the first yield point after `deadline_ns`
 * (CLOCK_MONOTONIC nanoseconds; 0 = none).  Yield points are between work items AND
 * inside one: a work item's batch is probed in slices of at most 1M rows
 * (mz_join_core.rs:862-934 yields inside a key group as well), each slice's results
 * consolidated and appended before the next starts. */
int32_t mzgpu_join_core_work_until(mzgpu_join* j, uint64_t fuel_rows, uint64_t deadline_ns, mzgpu_buf* out,
                                   int32_t* done);

/* --------------------------------------------------- a10: half_join */
/* dogs3 half_join_internal_unsafe as called at delta_join.rs:401-431: for each
 * stream update ((key, val1), time, d1) and each (key, val2, t, d2) in `trace`
 * with cmp(t, time): emit ((closure(key,val1,val2)), time, d1*d2).  The caller
 * must have advanced the trace's upper beyond every stream time (the operator
 * waits for the arrangement frontier in the reference).  Results are appended
 * to `out` (R32 rows, not consolidated unless consolidate_output != 0).
 * A probe sees at most 64 non-empty batches of `trace` (admitted layers plus
 * batches still waiting for physical compaction): advance the trace's physical
 * compaction (mzgpu_spine_set_physical_compaction) as the arrangement frontier
 * moves, as TraceManager::maintenance does, or the call returns
 * MZGPU_E_UNSUPPORTED once more than 64 batches have piled up. */
int32_t mzgpu_half_join(mzgpu_ctx* ctx, const mzgpu_r32* stream, uint64_t n, int32_t mem,
                        mzgpu_spine* trace, int32_t cmp_mode, const mzgpu_closure* closure,
                        int32_t consolidate_output, mzgpu_buf* out);
/* The same with the stream in a device buffer: nothing returns to the host. */
int32_t mzgpu_half_join_buf(mzgpu_ctx* ctx, mzgpu_buf* stream, mzgpu_spine* trace, int32_t cmp_mode,
                            const mzgpu_closure* closure, int32_t consolidate_output, mzgpu_buf* out);
/* k half joins over device-resident streams in one launch: the half-join stages that the delta
 * paths of one dataflow run side by side at a timestamp (`build_delta_join` renders one path per
 * input relation, delta_join.rs:71-310; their stages are independent operators).  Request j
 * probes streams[j] against traces[j] and appends to outs[j] exactly as
 * mzgpu_half_join_buf(..., consolidate_output = 0, ...) would; requests naming the same output
 * buffer must be adjacent and append in request order (the concatenation of the paths' outputs,
 * delta_join.rs:302-308).  closures may be NULL (identity closures for every request). */
int32_t mzgpu_half_join_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf* const* streams,
                             mzgpu_spine* const* traces, const int32_t* cmp_modes,
                             const mzgpu_closure* const* closures, mzgpu_buf* const* outs);
/* The first stage of k delta paths in one launch: request j forms the update stream of
 * batches[j] (build_update_stream, delta_join.rs:312-377: updates at skip_times[j] dropped unless
 * it is MZGPU_FRONTIER_EMPTY, initial_closures[j] applied) inside the probe kernel and half-joins
 * it against traces[j] -- the results of mzgpu_update_stream followed by mzgpu_half_join_buf(...,
 * consolidate_output = 0, ...) without materialising the stream.  Single-worker dataflows only:
 * with peers > 1 the stream is exchanged by its new key between the two steps. */
int32_t mzgpu_delta_first_stage_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_batch* const* batches,
                                     const mzgpu_closure* const* initial_closures, const uint64_t* skip_times,
                                     mzgpu_spine* const* traces, const int32_t* cmp_modes,
                                     const mzgpu_closure* const* closures, mzgpu_buf* const* outs);
/* build_update_stream (delta_join.rs:600-707): a batch's updates as a stream,
 * `initial_closure` applied (val2 unused), updates at `skip_time` dropped when
 * skip_time != MZGPU_FRONTIER_EMPTY (the as_of rule for source_relation != 0). */
int32_t mzgpu_update_stream(mzgpu_ctx* ctx, mzgpu_batch* batch, const mzgpu_closure* initial_closure,
                            uint64_t skip_time, mzgpu_buf* out);
/* Apply a closure to a stream of R32 rows (DeltaJoinFinalization / key-val
 * extraction of render_reduce, reduce.rs:106-157). */
int32_t mzgpu_map_rows(mzgpu_ctx* ctx, const mzgpu_r32* rows, uint64_t n, int32_t mem,
                       const mzgpu_closure* closure, mzgpu_buf* out);

/* ------------------------------------------- a11-a12: accumulable reduce */
/* build_accumulable (reduce.rs:1261-1471): state = the "ArrangeAccumulable"
 * arrangement (a spine of RACC batches). */
int32_t mzgpu_reduce_new(mzgpu_ctx* ctx, int32_t agg_kind, mzgpu_reduce** out);
/* A TopK operator (MZGPU_AGG_TOPK) behind the same handle: limit < 0 = no limit (LIMIT NULL),
 * offset >= 0, descending != 0 orders the values high to low.  Stepped with
 * mzgpu_reduce_accumulable[_buf] like every other kind. */
int32_t mzgpu_topk_new(mzgpu_ctx* ctx, int64_t limit, uint64_t offset, int32_t descending,
                       mzgpu_reduce** out);
void mzgpu_reduce_free(mzgpu_reduce* r);
/* One operator activation: `rows` are the (group key, value, time, diff)
 * updates with times in [previous upper, upper).  explode_one -> arrange ->
 * reduce_abelian: appends the output corrections (ROUT rows: -old, +new per
 * changed key and time) to `out`, consolidated. */
int32_t mzgpu_reduce_accumulable(mzgpu_reduce* r, const mzgpu_r32* rows, uint64_t n, int32_t mem,
                                 uint64_t upper, mzgpu_buf* out);
int32_t mzgpu_reduce_accumulable_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out);
/* The input arrangement (for sharing / inspection). Borrowed. */
mzgpu_spine* mzgpu_reduce_input_trace(mzgpu_reduce* r);

/* ---- accumulable reduce over several value columns ("lanes") in one arrangement
 * (build_accumulable over AccumulablePlan::simple_aggrs / full_aggrs, reduce.rs:1261-1471:
 * every input row explodes into one Accum per aggregate, arranged once, and reduce_abelian
 * emits one output row per key holding every finalized aggregate).  Lane l yields
 * COUNT(col_l) and SUM(col_l) exactly as the one-column kinds do; AVG is SUM / COUNT
 * downstream, and count(*) is any lane's count (NULLs are outside the fixed-width subset).
 *
 * A lane picks its column from the input row: field.src is MZGPU_SRC_VAL1 (R32 `val`, R40
 * `val1`) or MZGPU_SRC_VAL2 (R40 `val2`), field.shift / field.bits the bit-field
 * (dst_shift unused).  An I64 lane reads the field, sign-extended when sign_extend != 0
 * (a 64-bit field is the i64 itself); an F64 lane must pick a whole word (shift 0, bits 64). */
#define MZGPU_MAX_ACCUM_LANES 8
typedef struct mzgpu_accum_lane {
  int32_t kind;         /* MZGPU_AGG_COUNT_SUM_I64 or MZGPU_AGG_COUNT_SUM_F64, optionally | MZGPU_ACCUM_DISTINCT */
  uint32_t sign_extend; /* I64 lanes: sign-extend the bit-field                */
  mzgpu_field field;
} mzgpu_accum_lane;
/* OR'd into mzgpu_accum_lane.kind: the lane is COUNT(DISTINCT col) / SUM(DISTINCT col)
 * (AccumulablePlan::distinct_aggrs, src/compute-types/src/plan/reduce.rs:146-158; rendered by
 * build_accumulable, src/compute/src/render/reduce.rs:1338-1373).  Values are distinct by the lane's
 * i64 datum (after bit-field extraction and sign extension).  The operator keeps one more
 * arrangement per distinct lane, of R32 rows (group key, value, time, diff) keyed by the group key
 * (mzgpu_reduce_lanes_distinct_trace), and a (key, value) pair is present while its accumulated
 * multiplicity is non-zero -- a negative multiplicity counts as present, as in the reference, which
 * checks for errors only at the final arrangement.  Each change of presence adds one row to the
 * main arrangement: total = +-1 and only this lane's Accum, that of the value.  So a key's total
 * word is (number of plain lanes > 0 ? sum of the key's input diffs : 0) + the number of present
 * pairs over all distinct lanes, and that total decides the key's NULL-SUM and error flags as for
 * any lane.  Lane widths and classes do not change: a distinct lane is one lane of the class.
 *
 * MZGPU_AGG_COUNT_SUM_F64 | MZGPU_ACCUM_DISTINCT is MZGPU_E_UNSUPPORTED: whether the reference's
 * Row arrangement treats -0.0 / +0.0, and NaNs with different payloads, as one value depends on
 * the Row ordering versus Datum equality (src/repr/src/row.rs:1878-1881 and the tests near
 * :3768-3800), and nothing pins that here.  Any other bit in `kind` is MZGPU_E_INVALID. */
#define MZGPU_ACCUM_DISTINCT 0x100
/* Row widths.  The lane count rounds up to a class C in {1, 2, 4, 8}; the class's unused
 * lanes are zero.  Arrangement row: key, time, total, C x (non_nulls, acc_lo, acc_hi,
 * pos_infs, neg_infs, nans), padded to 16 bytes.  Output row: key, C x (count, sum_lo,
 * sum_hi), flags, time, diff, padded to 16 bytes (widths chosen so that no output width
 * equals an arrangement width: the generic kernels know a row by its width alone).
 *     C   arrangement          output
 *     1    80 B (mzgpu_racc)    64 B (mzgpu_rout)
 *     2   128 B                 96 B
 *     4   224 B                144 B
 *     8   416 B                240 B
 * Flags: bit 2l = lane l's SUM is NULL (total > 0 and the lane's accumulation is zero),
 * bit 2l+1 = lane l has net-zero records with a non-zero accumulation (the per-aggregate
 * AccumulableErrorCheck, reduce.rs:1418-1429).  A key has an output row while its whole
 * accumulated diff (total and every lane) is non-zero; a change in any lane retracts and
 * re-emits the whole row.  Output rows of C >= 2 are plain buffer rows:
 * mzgpu_buf_consolidate on them returns MZGPU_E_UNSUPPORTED (they leave the operator
 * consolidated).  The arrangement widths are accepted by batchers, builders and spines. */
#define MZGPU_ROW_RACC2 128
#define MZGPU_ROW_RACC4 224
#define MZGPU_ROW_RACC8 416
#define MZGPU_ROW_ROUT2 96
#define MZGPU_ROW_ROUT4 144
#define MZGPU_ROW_ROUT8 240
/* The arrangement and output row widths for n_lanes (1..8); MZGPU_E_INVALID otherwise. */
int32_t mzgpu_reduce_lanes_row_bytes(uint32_t n_lanes, uint32_t* arr_row_bytes, uint32_t* out_row_bytes);
/* in_row_bytes: 32 (R32) or 40 (R40), the rows the join operators emit.  A malformed
 * descriptor (kind, VAL2 on R32 input, a zero-width or out-of-range field, an F64 lane not
 * picking a whole word, n_lanes of 0 or above 8) is MZGPU_E_INVALID before any launch.
 * The handle is freed with mzgpu_reduce_free; mzgpu_reduce_input_trace returns its
 * arrangement. */
int32_t mzgpu_reduce_lanes_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                               uint32_t n_lanes, mzgpu_reduce** out);
/* One activation, with the protocol of mzgpu_reduce_accumulable[_buf]: `rows` are n input
 * rows of in_row_bytes with times in [previous upper, upper); the output corrections
 * (rows of the class's output width) are appended to `out`, consolidated.  After a failed
 * activation the operator reports that status from then on. */
int32_t mzgpu_reduce_lanes(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                           mzgpu_buf* out);
int32_t mzgpu_reduce_lanes_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out);
/* The pair arrangement of distinct lane `lane` (R32 rows: group key, value, time, diff; the
 * reference's "Arranged Accumulable Distinct"), borrowed like mzgpu_reduce_input_trace; NULL for a
 * lane without MZGPU_ACCUM_DISTINCT, a lane index out of range, or another operator. */
mzgpu_spine* mzgpu_reduce_lanes_distinct_trace(mzgpu_reduce* r, uint32_t lane);

/* ---- HAVING: the filter half of the reduce's fused mfp_after (render_reduce hands every reduce an
 * mfp_after, src/compute/src/render/reduce.rs:64-78; build_accumulable applies it to (key, finalized
 * aggregates) in its ReduceAccumulable closure, :1384-1409 and evaluate_mfp_after :1474-1499, and reports
 * its errors in AccumulableErrorCheck, :1452-1464).
 *
 * A filter is up to MZGPU_HAVING_MAX_PREDICATES predicates, evaluated in order as
 * SafeMfpPlan::evaluate_inner does (src/expr/src/linear.rs:1680-1700): the first predicate that is not
 * TRUE (FALSE or NULL) drops the row and later predicates are not evaluated; an error stops evaluation
 * with that error.  A predicate is a postfix program over typed values:
 *   INT   i64: a bit-field of the output key (optionally sign-extended, integer_to_bigint(#0{a}); a
 *         64-bit field is the i64 itself), a
 *         lane's COUNT, or an integer constant.  "int32" when it is a key field of at most 32 bits
 *         (sign-extended, or fewer than 32 bits), an integer constant in i32 range, or the result of
 *         a 32-bit operation.
 *   NUM   i128: the SUM of an int64 lane (numeric), or an i128 constant.
 *   FLOAT f64: the SUM of a float64 lane, or a constant.
 *   BOOL
 * A SUM is NULL when its lane's NULL flag (bit 2l) is set; a COUNT is never NULL.
 * Arithmetic is on INT only and carries its SQL width (arg = 32 or 64; a 32-bit operation takes int32
 * operands): add/sub/mul give NumericFieldOverflow when the result leaves the width
 * (src/expr/src/scalar/func.rs:107, 117, 690, 700, 904, 914); div truncates, a zero divisor gives
 * DivisionByZero and MIN / -1 Int32OutOfRange / Int64OutOfRange (func.rs:1037-1059).  Both operands
 * are evaluated; the first operand's error wins over the second's, and an error over a NULL, which
 * propagates (the eager argument unpacking of src/repr/src/scalar.rs:2126-2160).
 * Comparisons (arg = MZGPU_CMP_*, signed) take INT / INT, NUM / NUM, INT / NUM (the INT widened
 * exactly) or FLOAT / FLOAT, which compare as OrderedFloat (Datum::Float64, src/repr/src/scalar.rs:99:
 * NaN equals NaN and is above everything, -0.0 equals +0.0); a NULL operand gives NULL.
 * AND / OR / NOT are three-valued with the error rules of the variadic And / Or
 * (src/expr/src/scalar/func/variadic.rs:74-99, 1147-1170): for AND a FALSE operand wins over an
 * error, otherwise the larger error wins, otherwise NULL wins over TRUE; OR mirrors it with TRUE.
 *
 * Errors (in the order of the EvalError variants, src/expr/src/scalar.rs:1724-1740, which And's
 * std::cmp::max compares) are written into flag bits 16-18 of the output row
 * (MZGPU_ROUT_HAVING_ERR_SHIFT): this project carries errors as row flags, not in a separate error
 * collection.  A key has an output row at time t while its accumulated diff is non-zero (as without a
 * filter) AND it carries a lane error flag (bit 2l+1), or its predicates raised an error, or every
 * predicate is TRUE: error rows are never filtered away.  Corrections stay the (-old, +new) changes of
 * that visible row.  The map and project parts of mfp_after stay with the caller: the row layout does
 * not change, and a mapped column (SUM(b) + 1) is computed downstream; a map expression a predicate
 * reads (COUNT(b) + 1) is written inline in the predicate. */
#define MZGPU_HAVING_MAX_PREDICATES 4
#define MZGPU_HAVING_MAX_OPS 16 /* per predicate */
#define MZGPU_HAVING_MAX_CONSTS 8
#define MZGPU_HAVING_MAX_STACK 8
/* opcodes (mzgpu_having_op.code) */
#define MZGPU_HOP_KEY 1   /* push INT: bits [shift, shift + bits) of the key, sign-extended if sign_extend */
#define MZGPU_HOP_COUNT 2 /* push INT: COUNT of lane `arg` */
#define MZGPU_HOP_SUM 3   /* push SUM of lane `arg`: NUM (int64 lane) or FLOAT (float64 lane), NULL by flag 2l */
#define MZGPU_HOP_INT 4   /* push INT constant consts[konst] (in i64 range) */
#define MZGPU_HOP_NUM 5   /* push NUM constant consts[konst] */
#define MZGPU_HOP_FLOAT 6 /* push FLOAT constant: the f64 bits in consts[konst].lo */
#define MZGPU_HOP_ADD 7   /* INT, INT -> INT at width arg (32 or 64) */
#define MZGPU_HOP_SUB 8
#define MZGPU_HOP_MUL 9
#define MZGPU_HOP_DIV 10
#define MZGPU_HOP_CMP 11 /* arg = MZGPU_CMP_*: -> BOOL */
#define MZGPU_HOP_AND 12 /* BOOL, BOOL -> BOOL */
#define MZGPU_HOP_OR 13
#define MZGPU_HOP_NOT 14 /* BOOL -> BOOL */
/* the predicate error in flag bits 16-18 of an output row */
#define MZGPU_ROUT_HAVING_ERR_SHIFT 16
#define MZGPU_HAVING_ERR_DIVISION_BY_ZERO 1
#define MZGPU_HAVING_ERR_NUMERIC_FIELD_OVERFLOW 2
#define MZGPU_HAVING_ERR_INT32_OUT_OF_RANGE 3
#define MZGPU_HAVING_ERR_INT64_OUT_OF_RANGE 4
typedef struct mzgpu_having_op {
  uint8_t code;        /* MZGPU_HOP_* */
  uint8_t arg;         /* COUNT / SUM: lane; arithmetic: width 32 / 64; CMP: MZGPU_CMP_* */
  uint8_t shift;       /* KEY: right shift of the key word */
  uint8_t bits;        /* KEY: field width 1..64 */
  uint8_t sign_extend; /* KEY: sign-extend the field */
  uint8_t konst;       /* INT / NUM / FLOAT: constant index */
  uint8_t _pad[2];
} mzgpu_having_op;
typedef struct mzgpu_having_const {
  uint64_t lo, hi; /* INT / NUM: i128 two's complement; FLOAT: lo = the f64 bits, hi = 0 */
} mzgpu_having_const;
typedef struct mzgpu_having {
  uint32_t n_predicates; /* 0..MZGPU_HAVING_MAX_PREDICATES (0: no filter) */
  uint32_t n_consts;
  uint32_t n_ops[MZGPU_HAVING_MAX_PREDICATES];
  mzgpu_having_op ops[MZGPU_HAVING_MAX_PREDICATES][MZGPU_HAVING_MAX_OPS];
  mzgpu_having_const consts[MZGPU_HAVING_MAX_CONSTS];
} mzgpu_having;
/* mzgpu_reduce_lanes_new with a HAVING filter.  having == NULL, or n_predicates == 0, is exactly
 * mzgpu_reduce_lanes_new.  The lanes are checked first, as mzgpu_reduce_lanes_new does; the program is
 * then checked on the host, before any launch, and a program that fails leaves no operator behind (*out
 * is not written) and the context usable:
 * MZGPU_E_INVALID for a malformed one (unknown opcode, an empty predicate or more than
 * MZGPU_HAVING_MAX_OPS ops, stack underflow or a depth above MZGPU_HAVING_MAX_STACK, a lane >= n_lanes,
 * a bad key field, a bad width or compare op, a constant index >= n_consts, an INT constant outside
 * i64, an operand of the wrong type, a 32-bit operation on a value that is not int32, or a predicate
 * that does not leave exactly one BOOL); MZGPU_E_UNSUPPORTED for a well-formed program outside the
 * subset (arithmetic on a NUM or FLOAT, FLOAT compared with INT / NUM, BOOL compared with BOOL), so
 * that the caller keeps its own path at render time. */
int32_t mzgpu_reduce_lanes_new_having(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                                      uint32_t n_lanes, const mzgpu_having* having, mzgpu_reduce** out);

/* ---- monotonic MIN / MAX reduce: several MIN / MAX columns per key kept in the arrangement's diff
 * (HierarchicalPlan::Monotonic, src/compute-types/src/plan/reduce.rs:160-250, which the planner picks for
 * append-only inputs; rendered by build_monotonic, src/compute/src/render/reduce.rs:1138-1253).
 *
 * One activation:
 *   1. must_consolidate != 0: the rows are consolidated by (key, the lanes' values, time) first
 *      (consolidate_named_if): every value bit no lane reads is cleared, then equal rows fold, so a
 *      +1 / -1 pair at one time cancels.
 *   2. ensure_monotonic (src/timely-util/src/operator.rs:425-456): a row is kept iff its diff > 0.
 *      Every other row, diff == 0 included, is one error at its time: `errs` receives R16 rows
 *      (key = time, diff = rows rejected at that time), consolidated.  Rejected rows reach no key.
 *   3. A kept row's lane values become the diff, one Min / Max per lane; its multiplicity does not
 *      matter.  The arrangement keeps per (key, time) the per-lane extremum, and a key never leaves it
 *      once a row of it was kept (IsZero is always false).
 *   4. Output: per key, (key, the lanes' MIN / MAX) -- (-old, +new) whenever the accumulated values
 *      change, +new alone for the key's first kept row.
 *
 * Lanes reuse mzgpu_accum_lane: kind = MZGPU_AGG_MIN or MZGPU_AGG_MAX, field as for the lanes reduce
 * (src MZGPU_SRC_VAL1, or MZGPU_SRC_VAL2 of R40 input; shift, bits).  Unlike the accumulable lanes, where
 * a 64-bit field is always the i64, sign_extend chooses the ORDER here:
 *   sign_extend != 0: an int64 aggregate (MinInt16/32/64, MaxInt*, Date, Timestamp): the field
 *                     sign-extended, compared signed;
 *   sign_extend == 0: unsigned order (MinUInt*, MaxUInt*, MzTimestamp, Bool).
 * Output values are the natural values: the i64 bits of a signed lane, the u64 of an unsigned one.
 * NULLs are outside the fixed-width subset: every kept row carries a value for every lane.
 *
 * Lane word encoding in the arrangement (what mzgpu_reduce_input_trace exports): word = value
 * ^ 2^63 for a signed lane, complemented on top of that for MIN, so every lane accumulates as an
 * unsigned MAX and zero is the identity.  The same xor decodes a word.
 *
 * Row widths (lane count rounds up to a class of 4 or 8; unused lanes are zero):
 *     lanes   arrangement                                   output
 *     1-4      48 B: key, time | 4 lane words                56 B: key, 4 values, time, diff
 *     5-8     112 B: key, time | 8 lane words, 4 zero words  88 B: key, 8 values, time, diff
 * The output rows have no generic meaning: mzgpu_buf_consolidate on them returns MZGPU_E_UNSUPPORTED
 * (they leave the operator consolidated).  The arrangement widths are accepted by batchers, builders and
 * spines, and accumulate there by the per-word max.
 *
 * Not supported: float64 MIN / MAX (OrderedFloat ties -0.0 with +0.0, and NaNs with different payloads,
 * so which bits survive would depend on arrival order), HAVING on this operator, and COUNT / SUM in the same operator (a MonotonicPlan holds MIN / MAX-type functions
 * only). */
/* OR'd into a MIN / MAX lane's kind: the column is float64.  Always MZGPU_E_UNSUPPORTED (see above), so
 * that a caller describing such a plan keeps its own path. */
#define MZGPU_MONO_F64 0x200
#define MZGPU_ROW_RMONO4 48
#define MZGPU_ROW_RMONO8 112
#define MZGPU_ROW_MONO_OUT4 56
#define MZGPU_ROW_MONO_OUT8 88
/* The arrangement and output row widths for n_lanes (1..8); MZGPU_E_INVALID otherwise. */
int32_t mzgpu_reduce_monotonic_row_bytes(uint32_t n_lanes, uint32_t* arr_row_bytes, uint32_t* out_row_bytes);
/* in_row_bytes: 32 (R32) or 40 (R40); n_lanes 1..8.  Checked on the host before any launch:
 * MZGPU_E_INVALID for a malformed descriptor (a kind other than MIN / MAX, a COUNT / SUM kind, any flag bit
 * but MZGPU_MONO_F64, VAL2 on R32 input, a zero-width or out-of-range field, n_lanes of 0 or above 8);
 * then MZGPU_E_UNSUPPORTED for a float64 lane.  A failure leaves no operator behind (*out is not written)
 * and the context usable.  The handle is freed with mzgpu_reduce_free; mzgpu_reduce_input_trace returns its
 * arrangement. */
int32_t mzgpu_reduce_monotonic_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                                   uint32_t n_lanes, int32_t must_consolidate, mzgpu_reduce** out);
/* One activation, with the protocol of mzgpu_reduce_lanes[_buf]: `rows` are n input rows of
 * in_row_bytes with times in [previous upper, upper); the corrections (rows of the class's output width)
 * are appended to `out`, consolidated, and the errors (R16) to `errs` (required).  After a failed
 * activation the operator reports that status from then on. */
int32_t mzgpu_reduce_monotonic(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                               mzgpu_buf* out, mzgpu_buf* errs);
int32_t mzgpu_reduce_monotonic_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out,
                                   mzgpu_buf* errs);

/* ---- hierarchical MIN / MAX reduce: several MIN / MAX columns per key over input with retractions, one output
 * row per key (HierarchicalPlan::Bucketed with several aggr_funcs, BucketedPlan in
 * src/compute-types/src/plan/reduce.rs:232-250, which the planner picks for MIN / MAX over any collection that can
 * retract; rendered by build_bucketed / build_bucketed_negated_output, src/compute/src/render/reduce.rs:796-1135).
 *
 * Lanes reuse mzgpu_accum_lane exactly as mzgpu_reduce_monotonic_new does: kind = MZGPU_AGG_MIN or MZGPU_AGG_MAX,
 * sign_extend chooses signed or unsigned order, field picks the bit-field (src MZGPU_SRC_VAL1, or MZGPU_SRC_VAL2 of
 * R40 input).  MZGPU_MONO_F64 is MZGPU_E_UNSUPPORTED for the same OrderedFloat reason.  Input is R32 or R40 rows.
 *
 * Per key, at every time t, the key's live multiset is its input rows with times <= t, each masked to the value
 * bits some lane reads and consolidated by (key, masked val1, masked val2) -- the reference arranges (key, row of
 * the aggregates' inputs), so two rows that differ only in bits no lane reads are one value row and a +1 / -1 pair
 * of them cancels.  Then:
 *   every live count positive: the key's output row holds, per lane, the MIN / MAX of its field over the live
 *       rows (the natural values, as the monotonic operator emits them);
 *   some live count negative ("non-positive accumulation"): no output row while the key is in that state, and one
 *       error for it;
 *   no live row: no output row.
 * Output (`out`): rows of the monotonic output widths, MZGPU_ROW_MONO_OUT4 (56 B, 1-4 lanes) or
 *     MZGPU_ROW_MONO_OUT8 (88 B, 5-8 lanes): key, the C values (unused lanes zero), time, diff.  A change in any lane
 *     emits (-old, +new) at the time of the change.  The rows leave the operator consolidated and sorted per key.
 * Errors (`errs`, R32 rows (key, 0, time, diff), consolidated): +1 when a key enters the non-positive state at
 *     time t, -1 when it leaves it.  This is a fixed-width stand-in for the reference's per-key error "saw
 *     non-positive accumulation for key ... in hierarchical mins-maxes aggregate"; the reference's ok output for such
 *     a key depends on how its buckets hash, and is deliberately not reproduced.
 * State: mzgpu_reduce_input_trace(r) returns the operator's arrangement: the masked input rows at the input width
 *     (R32 or R40) with ordinary SUM diffs.  The caller compacts it like any other trace.  Work per touched key is
 *     its distinct live value rows while they fit a 32-entry table, and one ordered pass over its runs per new time
 *     beyond that.
 * Checked on the host before any launch, in the order of mzgpu_reduce_monotonic_new: MZGPU_E_INVALID for a
 * malformed descriptor (in_row_bytes not 32 / 40, a kind other than MIN / MAX, any flag bit but MZGPU_MONO_F64, VAL2
 * on R32 input, a zero-width or out-of-range field, n_lanes of 0 or above 8), then MZGPU_E_UNSUPPORTED for a float64
 * lane.  A failure leaves no operator behind (*out is not written) and the context usable.  The handle is freed with
 * mzgpu_reduce_free.
 * Not supported: COUNT / SUM lanes in the same operator (ReducePlan::Collation: a caller zips this operator's output
 * with mzgpu_reduce_lanes_new's by key), HAVING on MIN / MAX, float64 lanes, NULLs, and the bucket tree itself. */
int32_t mzgpu_reduce_hierarchical_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                                      uint32_t n_lanes, mzgpu_reduce** out);
/* One activation, with the protocol of mzgpu_reduce_monotonic[_buf]: `rows` are n input rows of in_row_bytes with
 * times in [previous upper, upper); the corrections (rows of the class's output width) are appended to `out` and
 * the errors (R32) to `errs` (required).  After a failed activation the operator reports that status from then
 * on. */
int32_t mzgpu_reduce_hierarchical(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                                  mzgpu_buf* out, mzgpu_buf* errs);
int32_t mzgpu_reduce_hierarchical_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out,
                                      mzgpu_buf* errs);

/* ---- monotonic TopK: Top-1 and Top-K over append-only input, with only the window arranged
 * (TopKPlan::MonotonicTop1 / MonotonicTopK, src/compute/src/render/top_k.rs:102-214; the planner picks them
 * for every offset-0 TopK over an append-only input, src/compute-types/src/plan/top_k.rs:47-92).  One operator
 * covers both: Top1 is limit = 1, the same collection and the same one-row-per-key state.
 *
 * Input: R32 or R40 rows; `key` is the group key and the row is (key, val1[, val2]).
 * Order: rows of a key compare by the order lanes in sequence (the plan's order_key; n_order = 0 is no ORDER
 * BY).  A lane's field is sign-extended and compared signed when sign_extend != 0, unsigned otherwise, and
 * reversed when descending.  Rows equal on every lane are ordered by val1, then val2, as unsigned words:
 * the fixed-width stand-in for compare_columns(order_key, l, r, || l.cmp(r)) (Top1Monoid,
 * top_k.rs:866-932), which breaks ties by the whole row's Datum order.  The two agree when every column the
 * plan can tie on is listed as a lane, or when signed columns are encoded with the sign bit flipped (then
 * the unsigned word order is the Datum order).
 *
 * One activation, as build_monotonic's steps:
 *   1. must_consolidate != 0: the rows are consolidated by the whole row, then time (consolidate_named_if,
 *      top_k.rs:446-511).
 *   2. ensure_monotonic (src/timely-util/src/operator.rs:425-456): a row is kept iff its diff > 0.  Every
 *      other row is one error at its time: `errs` receives R16 rows (key = time, diff = rows rejected at that
 *      time), consolidated, as mzgpu_reduce_monotonic does.
 *   3. A kept row's multiplicity counts toward the limit (TopKBatch, top_k.rs:765-850): a limit can cut
 *      inside one row's copies, and Top1 always yields diff 1 (top_k.rs:564).
 *   4. Output: rows of the INPUT width appended to `out`, consolidated and sorted: (key, val1[, val2], time,
 *      diff), diff the change of that row's multiplicity inside the window.  At every time the window is the
 *      first `limit` units per key of the accumulated kept input, in the order above (the TopK the
 *      reference's thinning, topk stage and delayed retraction feedback, top_k.rs:116-214, compute).
 *      They are ordinary R32 / R40 rows.
 * State: mzgpu_reduce_input_trace(r) returns the window arrangement, MZGPU_ROW_RTOPK rows
 *     (key, o0, o1, o2, val1, val2, time | diff, pad), o_j the encoded lane j: the field (sign-extended
 * when signed) ^ 2^63 if signed, complemented if descending; unused words and val2 of R32 input are 0.  The
 * caller compacts it like any other trace; after logical compaction and merges it holds exactly the live
 * window, at most `limit` units per key.  Work per touched key is bounded by its live window plus its
 * not-yet-compacted rows, not by its history.
 * limit: >= 0; MZGPU_TOPK_NO_LIMIT is LIMIT NULL / None (Diff::MAX, top_k.rs:564, :721): every kept row enters
 * and no state is read.
 * Checked on the host before any launch; a failure leaves no operator behind and the context usable:
 *   MZGPU_E_INVALID: in_row_bytes not 32 / 40, VAL2 on R32 input, a zero-width or out-of-range field, unknown
 *       flag bits, n_order > MZGPU_MAX_ORDER_LANES, or a NULL `order` with n_order > 0;
 *   MZGPU_E_UNSUPPORTED: a float64 order lane (MZGPU_ORDER_F64: OrderedFloat ties -0.0 with +0.0 and NaN
 *       payloads), or a negative limit (the reference's NegLimit error path, top_k.rs:67-98).
 * Not supported: offset > 0 (never planned as monotonic), limit expressions (INTEGRATION.md), NULLs. */
typedef struct mzgpu_order_lane { /* one ColumnOrder of the plan's order_key */
  uint32_t sign_extend;           /* != 0: signed order of the sign-extended field */
  uint32_t descending;            /* ColumnOrder::desc */
  uint32_t flags;                 /* 0, or MZGPU_ORDER_F64 */
  mzgpu_field field;              /* src MZGPU_SRC_VAL1, or MZGPU_SRC_VAL2 of R40 input; shift; bits */
} mzgpu_order_lane;
#define MZGPU_ORDER_F64 0x1 /* the column is float64: always MZGPU_E_UNSUPPORTED */
#define MZGPU_MAX_ORDER_LANES 3
#define MZGPU_TOPK_NO_LIMIT INT64_MAX
#define MZGPU_ROW_RTOPK 72
int32_t mzgpu_topk_monotonic_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_order_lane* order,
                                 uint32_t n_order, int64_t limit, int32_t must_consolidate, mzgpu_reduce** out);
/* One activation, with the protocol of mzgpu_reduce_monotonic[_buf]: `rows` are n input rows with times in
 * [previous upper, upper); the window changes (input-width rows) are appended to `out`, the errors (R16) to
 * `errs` (required).  After a failed activation the operator reports that status from then on. */
int32_t mzgpu_topk_monotonic(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                             mzgpu_buf* out, mzgpu_buf* errs);
int32_t mzgpu_topk_monotonic_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out, mzgpu_buf* errs);

/* ---- basic TopK: whole rows over input with retractions, up to three order columns, OFFSET
 * (TopKPlan::Basic, which the planner picks for every TopK that is not monotonic: input that retracts, such as
 * a join's output, and every TopK with an OFFSET, src/compute-types/src/plan/top_k.rs:47-92; rendered by
 * build_topk / build_topk_stage / build_topk_negated_stage, src/compute/src/render/top_k.rs:215-444, 521-673).
 *
 * Input: R32 or R40 rows with any diffs; `key` is the group key and the row is (key, val1[, val2]).
 * Order: as for mzgpu_topk_monotonic_new (the same mzgpu_order_lane, 0 to 3 lanes, each signed or unsigned
 * and possibly descending).  Rows equal on every lane are ordered by val1, then val2, as unsigned words: the
 * fixed-width stand-in for compare_columns(order_key, l, r, || l.cmp(r)), which breaks ties by the whole row's
 * Datum order.  The two agree when every column the plan can tie on is listed as a lane, or when signed columns
 * are encoded with the sign bit flipped (then the unsigned word order is the Datum order).
 *
 * Per key, at every time t, the key's live rows are its input rows with times <= t consolidated by
 * (key, val1, val2).  Then:
 *   every live count positive: the window is the units in positions [offset, offset + limit) of the ordered
 *       multiset, counting multiplicities, so a limit or an offset can cut inside one row's copies (as
 *       build_topk_negated_stage does, top_k.rs:605-669);
 *   some live count negative (the reference's "Negative multiplicities in TopK"): the key is in the error state
 *       and has no window;
 *   no live row: no window.
 * Output (`out`): rows of the INPUT width, (key, val1[, val2], time, diff), diff the change of that row's
 *     multiplicity inside the window, consolidated and sorted per key: the collection the reference builds as
 *     input.concat(negated_output).
 * Errors (`errs`, R32 rows (key, 0, time, diff), consolidated): +1 when a key enters the error state at time t,
 *     -1 when it leaves it.  This is the fixed-width stand-in that mzgpu_reduce_hierarchical_new uses; the
 *     reference's ok output for such a key depends on how its buckets hash, and is deliberately not reproduced.
 * State:
 *   mzgpu_reduce_input_trace(r) returns the whole live input, one MZGPU_ROW_RTOPK row per input row (encoded
 *       as for mzgpu_topk_monotonic_new) with ordinary SUM diffs.  The caller compacts it like any other trace.
 *   mzgpu_topk_basic_negatives_trace(r) returns the negatives arrangement (borrowed, for inspection and size
 *       logging): R32 rows (key, 0, time, delta) whose deltas, summed over a key, count that key's rows with a
 *       negative accumulated count.  The operator advances its logical and physical compaction to `upper` after
 *       each activation, so after merges it holds about one row per key in the error state.
 * Work per touched key and new time: its window prefix (its rows up to unit offset + limit, plus cancelled rows
 *     not yet compacted), plus its new rows, plus one binary search per prior batch per touched row.  It does not
 *     depend on the group's size, with one exception: a key entering or leaving the error state under LIMIT NULL
 *     emits its whole window.
 * limit: >= 0; MZGPU_TOPK_NO_LIMIT is LIMIT NULL / None.  offset: OFFSET, any value.
 * Checked on the host before any launch; a failure leaves no operator behind and the context usable:
 *   MZGPU_E_INVALID: everything mzgpu_topk_monotonic_new refuses as invalid;
 *   MZGPU_E_UNSUPPORTED: a float64 order lane, a negative limit (the reference's NegLimit path), or
 *       offset + limit past INT64_MAX with a finite limit (the reference then makes the limit an expression,
 *       top_k.rs:284-303).
 * Not supported: limit expressions, NULLs, float64 order columns, and the bucket tree itself (the negatives
 * arrangement is what bounds the work instead). */
int32_t mzgpu_topk_basic_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_order_lane* order, uint32_t n_order,
                             int64_t limit, uint64_t offset, mzgpu_reduce** out);
/* One activation, with the protocol of mzgpu_reduce_hierarchical[_buf]: `rows` are n input rows with times in
 * [previous upper, upper); the window changes (input-width rows) are appended to `out`, the errors (R32) to
 * `errs` (required; not `out`).  After a failed activation the operator reports that status from then on. */
int32_t mzgpu_topk_basic(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper, mzgpu_buf* out,
                         mzgpu_buf* errs);
int32_t mzgpu_topk_basic_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out, mzgpu_buf* errs);
mzgpu_spine* mzgpu_topk_basic_negatives_trace(mzgpu_reduce* r); /* borrowed, for inspection and size logging */

/* ---- temporal filters: the device MfpPlan (src/expr/src/linear.rs:1730-1990), with the updates it produces at
 * future times held in a bucket chain until the frontier reaches them (the temporal delay operator,
 * src/compute/src/extensions/temporal_bucket.rs, over BucketChain, src/timely-util/src/temporal.rs:59-211).
 *
 * Input: R32 or R40 rows with any diffs.  Output: R32 or R40 rows whose words (key, val1 and, for R40, val2)
 * are each an OR of up to MZGPU_MAX_FIELDS bit-fields (mzgpu_field, src MZGPU_SRC_KEY / VAL1 / VAL2, where
 * VAL2 is the R40 input's second value word, or MZGPU_SRC_MAP(i), map expression i of mzgpu_mfp_new_map).
 *
 * Non-temporal predicates (0..MZGPU_MFP_MAX_PREDICATES) are programs of the HAVING interpreter
 * (mzgpu_having_op; same types, width rules, errors and three-valued AND / OR / NOT) evaluated in order as
 * SafeMfpPlan::evaluate_inner does: the first one that is not TRUE drops the row; an error stops evaluation
 * and becomes an error update at the row's (time, diff).  The one difference: MZGPU_HOP_COL (the HAVING
 * opcode MZGPU_HOP_KEY) pushes a bit-field of source word `arg` (MZGPU_SRC_*) instead of the key.
 * MZGPU_HOP_COUNT / SUM / NUM / FLOAT are MZGPU_E_INVALID here.  No value is NULL: nullable columns are
 * outside the fixed-width subset.
 *
 * Temporal predicates (0..MZGPU_MFP_MAX_TEMPORAL) read `mz_now() CMP expr` with CMP one of MZGPU_CMP_EQ / LT /
 * LE / GT / GE; expr is a program that leaves one MZTS (u64 mz_timestamp).  The bound lists are derived as
 * MfpPlan::create_from does (linear.rs:1772-1804), in predicate order: EQ adds expr to the lower bounds and
 * step_mz_timestamp(expr) to the upper bounds, LT adds expr to the upper bounds, LE adds step(expr) to them,
 * GT adds step(expr) to the lower bounds and GE adds expr to them.  step_mz_timestamp(u64::MAX) is
 * MzTimestampStepOverflow.  Beyond the integer ops a temporal program has:
 *   MZGPU_HOP_COL_MZTS     push MZTS: the unsigned bit-field of word `arg` (uint8_to_mz_timestamp, an
 *                          mz_timestamp column); cannot fail
 *   MZGPU_HOP_INT_TO_MZTS  INT -> MZTS (bigint / integer_to_mz_timestamp); a negative value is
 *                          MzTimestampOutOfRange with the value as payload
 *   MZGPU_HOP_COL_TS       push TS: a `timestamp` column, the (sign-extended) field as i64 microseconds
 *                          since 1970-01-01 00:00:00
 *   MZGPU_HOP_COL_DATE     push DATE: a `date` column, the (sign-extended) field as i32 days since 1970-01-01
 *   MZGPU_HOP_TS_ADD_IV    TS + the constant interval consts[konst] (lo = microseconds as i64, hi = days in
 *                          bits 0-31 and months in bits 32-63, both i32); a result outside
 *                          [LOW_DATE, HIGH_DATE] = [-4713-12-31, 262142-12-31] is TimestampOutOfRange
 *                          (add_timestamplike_interval, src/expr/src/scalar/func.rs:200-213)
 *   MZGPU_HOP_TS_TO_MZTS   TS -> MZTS: milliseconds, rounded toward -inf (timestamp_millis); a negative
 *                          result is MzTimestampOutOfRange with the microseconds as payload
 *   MZGPU_HOP_DATE_TO_MZTS DATE -> MZTS: days * 86,400,000; a negative result is MzTimestampOutOfRange with
 *                          the days as payload
 * MZTS, TS and DATE values are MZGPU_E_UNSUPPORTED in a non-temporal predicate: it keeps payload-carrying
 * errors out of AND / OR, whose order would compare error strings.
 *
 * Per input row (time, diff), exactly MfpPlan::evaluate (linear.rs:1865-1971), with valid(t) = t < until
 * (until = MZGPU_FRONTIER_EMPTY: every time is valid):
 *   the predicates; then lower = max(time, every lower bound), evaluated in order, the first error wins; a
 *   row whose lower is not valid is dropped before any upper bound is evaluated; upper = the minimum of the
 *   upper bounds, clamped to at least lower, and evaluation stops once upper == lower (later upper-bound
 *   errors are never raised); an invalid upper becomes "none"; if lower != upper the output gets
 *   (row, lower, +diff) and, if there is an upper, (row, upper, -diff).
 * Errors are R32 rows (code, payload, time, diff) in `errs`, consolidated.  The codes are numbered in the
 * order of the EvalError variants (src/expr/src/scalar.rs:1724-1750): the four HAVING codes, then
 * MZGPU_MFP_ERR_MZ_TIMESTAMP_OUT_OF_RANGE (payload: the operand, as the reference's message embeds it),
 * MZGPU_MFP_ERR_MZ_TIMESTAMP_STEP_OVERFLOW and MZGPU_MFP_ERR_TIMESTAMP_OUT_OF_RANGE (payload 0).
 *
 * mzgpu_mfp_step(op, rows, upper, out, errs): evaluates the new rows and appends to `out` every resulting
 * update with time < upper together with every held update that has become due, consolidated (the
 * project's consolidated row order), and appends the errors to `errs`.  Everything else is held.  `upper`
 * must not decrease (MZGPU_E_FRONTIER).  upper == MZGPU_FRONTIER_EMPTY ("no more times") releases everything,
 * time u64::MAX included.  The _buf form reads rows and their count from the device and returns nothing to
 * the host (beyond what consolidating a release whose bound exceeds the fused kernel's limit reads back).
 *
 * Row counts stay on the device: a step's buffers are sized by host bounds (2 updates per new row; a held
 * slice by its segment's bound until the segment's header has been read back, which happens asynchronously and
 * never blocks a step).  Held updates live in a bucket chain: buckets [start, start + 2^bits) covering [upper, 2^64), each owning
 * device row segments.  A step inserts its held rows with one partition pass over at most 64 bucket bounds
 * (a histogram and a scatter, no sort; a step's held rows are inserted at the start of the next step, or by
 * mzgpu_mfp_frontier / mzgpu_mfp_stats, once their count is known), peels the buckets below `upper` and splits the
 * one that straddles it
 * (a two-way time partition), then restores the chain (adjacent buckets within two bits of each other)
 * with fuel counted in rows, MZGPU_MFP_RESTORE_FUEL per step (temporal_bucket.rs:159-165).
 *
 * mzgpu_mfp_frontier(op, &t): t = the least held time, or MZGPU_FRONTIER_EMPTY when nothing is held: where the
 * caller holds its capability, as the delay operator does.  On any other status t is not written (a failed
 * read must not look like "nothing held").  mzgpu_mfp_stats(op, out): out[0] = held rows, out[1] = buckets,
 * out[2] = rows the store read and wrote in the last step (insert, peel, splits and restore; the new rows'
 * evaluation and the release's consolidation are not store work).  Both wait for the device.
 *
 * Refused on the host before any launch (no operator is created and the context stays usable):
 * MZGPU_E_INVALID for a malformed plan (row widths, projection fields, predicate / temporal / op / constant
 * counts, unknown opcodes or compare ops, stack underflow or overflow, operand types, a program that does
 * not leave one BOOL / one MZTS); MZGPU_E_UNSUPPORTED for a well-formed plan outside the subset (an interval
 * with months, or whose days and microseconds leave i64 microseconds; MZTS / TS / DATE in a non-temporal
 * predicate; a float64 column, MZGPU_HOP_COL_F64), so that the caller keeps the Rust operator at render time. */
#define MZGPU_MFP_MAX_PREDICATES 4
#define MZGPU_MFP_MAX_TEMPORAL 4
#define MZGPU_MFP_MAX_OPS 16 /* per program */
#define MZGPU_MFP_MAX_CONSTS 8
#define MZGPU_MFP_RESTORE_FUEL 1000000
#define MZGPU_HOP_COL MZGPU_HOP_KEY /* push INT: bits [shift, shift + bits) of source word arg */
#define MZGPU_HOP_COL_MZTS 15
#define MZGPU_HOP_INT_TO_MZTS 16
#define MZGPU_HOP_COL_TS 17
#define MZGPU_HOP_COL_DATE 18
#define MZGPU_HOP_TS_ADD_IV 19
#define MZGPU_HOP_TS_TO_MZTS 20
#define MZGPU_HOP_DATE_TO_MZTS 21
#define MZGPU_HOP_COL_F64 22 /* a float64 column (word arg): always MZGPU_E_UNSUPPORTED */
#define MZGPU_MFP_ERR_MZ_TIMESTAMP_OUT_OF_RANGE 5
#define MZGPU_MFP_ERR_MZ_TIMESTAMP_STEP_OVERFLOW 6
#define MZGPU_MFP_ERR_TIMESTAMP_OUT_OF_RANGE 7
typedef struct mzgpu_mfp {
  uint32_t in_row_bytes;  /* 32 or 40 */
  uint32_t out_row_bytes; /* 32 or 40 */
  uint32_t n_fields[3];   /* fields of the output key, val1, val2 (val2: R40 output only) */
  mzgpu_field fields[3][MZGPU_MAX_FIELDS];
  uint32_t n_predicates;
  uint32_t n_temporal;
  uint32_t n_consts;
  uint32_t temporal_cmp[MZGPU_MFP_MAX_TEMPORAL]; /* MZGPU_CMP_EQ / LT / LE / GT / GE */
  uint32_t n_ops[MZGPU_MFP_MAX_PREDICATES];
  uint32_t n_temporal_ops[MZGPU_MFP_MAX_TEMPORAL];
  mzgpu_having_op ops[MZGPU_MFP_MAX_PREDICATES][MZGPU_MFP_MAX_OPS];
  mzgpu_having_op temporal_ops[MZGPU_MFP_MAX_TEMPORAL][MZGPU_MFP_MAX_OPS];
  mzgpu_having_const consts[MZGPU_MFP_MAX_CONSTS];
} mzgpu_mfp;
typedef struct mzgpu_mfp_op mzgpu_mfp_op;
int32_t mzgpu_mfp_new(mzgpu_ctx* ctx, const mzgpu_mfp* plan, uint64_t until, mzgpu_mfp_op** out);

/* ---- map expressions of the device MfpPlan: the `expressions` of a MapFilterProject, computed per row, read by
 * the predicates and the temporal bounds and projected into the output (SafeMfpPlan::evaluate_inner,
 * src/expr/src/linear.rs:1680-1700).
 *
 * mzgpu_mfp_new_map(ctx, plan, map, until, out) is mzgpu_mfp_new with map->n_exprs expressions appended to the
 * input columns; map == NULL or n_exprs == 0 is exactly mzgpu_mfp_new (which is that call).  Each expression is a
 * postfix program of the same interpreter that leaves one value of any type (INT, BOOL, MZTS, TS or DATE); its
 * constants index map->consts, not plan->consts.  The opcodes beyond those of the predicates:
 *   MZGPU_HOP_MAP arg         push the value of expression `arg`, with its type.  Inside expression i only
 *                             arg < i; predicates and temporal programs may read any expression
 *   MZGPU_HOP_NEG / ABS       INT -> INT at width arg (neg_int32/64, abs_int32/64): the width's minimum is
 *                             Int32OutOfRange / Int64OutOfRange with the operand as payload
 *   MZGPU_HOP_MOD             INT, INT -> INT at width arg (mod_int32/64): a zero divisor is DivisionByZero,
 *                             MIN % -1 is 0
 *   MZGPU_HOP_INT64_TO_INT32  INT -> int32 (cast_int64_to_int32): out of range is Int32OutOfRange with the
 *                             operand as payload
 *   MZGPU_HOP_IF              BOOL, T, T -> T (MirScalarExpr::If; both branches of one type, or both INT): an
 *                             error in the condition is the result, otherwise the taken branch's value or error;
 *                             an error in the branch not taken never surfaces
 * A MZGPU_HOP_MAP value never carries an error: an expression's error stops the row before anything reads it.
 * AND / OR do not take an operand that may carry an error whose payload varies with the data (from
 * MZGPU_HOP_INT64_TO_INT32 or an mz_timestamp cast): the reference orders two such errors by their message
 * strings.  Such a program is MZGPU_E_UNSUPPORTED.  When AND / OR meet two errors of one code, the payload-0 one
 * (a division's "a / b" message) wins over NEG / ABS's operand, as the longer string does.
 *
 * Per input row, in the order of SafeMfpPlan::evaluate_inner and MfpPlan::evaluate:
 *   1. the support of predicate p is 1 + the highest MZGPU_HOP_MAP index it reads (0 if none);
 *   2. before p runs, the expressions not yet evaluated below its support are evaluated in index order; an
 *      expression error stops the row and becomes an error update at the row's (time, diff); a predicate that is
 *      not TRUE drops the row;
 *   3. once every predicate has passed, every remaining expression is evaluated, projected or not: its errors
 *      count;
 *   4. the temporal bounds are evaluated as for mzgpu_mfp_new, and may read expressions (MZTS-typed ones);
 *   5. the output row is the projection over the input words and the expression values: a field with src
 *      MZGPU_SRC_MAP(i) takes bits [shift, shift + bits) of expression i's value (an INT as two's-complement
 *      i64, a BOOL as 0 / 1, an MZTS, TS or DATE as its u64 bits).
 * Errors are the R32 error rows of mzgpu_mfp_new with its codes.
 *
 * Refused on the host before any launch, leaving no operator and the context usable: MZGPU_E_INVALID for a
 * forward MZGPU_HOP_MAP reference, type errors, a wrong stack depth, more than MZGPU_MFP_MAX_MAPS expressions,
 * MZGPU_MFP_MAX_OPS ops or MZGPU_MFP_MAX_CONSTS constants, and a projected expression index >= n_exprs;
 * MZGPU_E_UNSUPPORTED for everything mzgpu_mfp_new refuses as unsupported (MZTS / TS / DATE values in a
 * non-temporal predicate, which includes an expression of those types read by one) and the AND / OR rule above.
 * Not supported: float64 columns and arithmetic, numeric, NULLs, variable-width values.  Step, frontier, stats
 * and free are those of mzgpu_mfp_new. */
#define MZGPU_MFP_MAX_MAPS 8
#define MZGPU_SRC_MAP0 16 /* mzgpu_field.src of expression 0 (above every MZGPU_SRC_*) */
#define MZGPU_SRC_MAP(i) (MZGPU_SRC_MAP0 + (i))
#define MZGPU_HOP_MAP 23
#define MZGPU_HOP_NEG 24
#define MZGPU_HOP_ABS 25
#define MZGPU_HOP_MOD 26
#define MZGPU_HOP_INT64_TO_INT32 27
#define MZGPU_HOP_IF 28
typedef struct mzgpu_mfp_map {
  uint32_t n_exprs; /* 0..MZGPU_MFP_MAX_MAPS */
  uint32_t n_consts;
  uint32_t n_ops[MZGPU_MFP_MAX_MAPS];
  mzgpu_having_op ops[MZGPU_MFP_MAX_MAPS][MZGPU_MFP_MAX_OPS];
  mzgpu_having_const consts[MZGPU_MFP_MAX_CONSTS];
} mzgpu_mfp_map;
int32_t mzgpu_mfp_new_map(mzgpu_ctx* ctx, const mzgpu_mfp* plan, const mzgpu_mfp_map* map, uint64_t until,
                          mzgpu_mfp_op** out);
void mzgpu_mfp_free(mzgpu_mfp_op* op);
int32_t mzgpu_mfp_step(mzgpu_mfp_op* op, const void* rows, uint64_t n, int32_t mem, uint64_t upper, mzgpu_buf* out,
                       mzgpu_buf* errs);
int32_t mzgpu_mfp_step_buf(mzgpu_mfp_op* op, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out, mzgpu_buf* errs);
int32_t mzgpu_mfp_frontier(mzgpu_mfp_op* op, uint64_t* out);
int32_t mzgpu_mfp_stats(mzgpu_mfp_op* op, uint64_t out[3]);

/* ---- join closures: the device MfpPlan as the closure of the probe operators (JoinClosure,
 * src/compute-types/src/plan/join.rs:50-82, applied by every half join, delta_join.rs:383-591, and every join_core
 * stage of a linear join, linear_join.rs:460-500).
 *
 * mzgpu_join_closure_new(ctx, plan, map, out) checks the plan once, with the validation and plan build of
 * mzgpu_mfp_new_map, and keeps it in device memory.  The plan reads three input words: plan->in_row_bytes is 40,
 * source word MZGPU_SRC_KEY is the key, MZGPU_SRC_VAL1 the stream row's value and MZGPU_SRC_VAL2 the lookup row's
 * value (for join_core: trace1's value and trace2's value, whichever side pushed).  out_row_bytes is 32 or 40.
 * Predicates, map expressions, projection, types, error codes and error order are those of mzgpu_mfp_new_map.
 * Refused, leaving no handle and the context usable: in_row_bytes != 40 and n_temporal != 0 (a JoinClosure's plan
 * is a SafeMfpPlan) with MZGPU_E_INVALID, and everything mzgpu_mfp_new_map refuses, with its status.  A join or
 * a call using the handle must not outlive it.
 *
 * ready_equivalences are lowered by the caller into leading predicates: a class [e0, e1, ..., en] becomes
 * CMP_EQ(e0, e1), ..., CMP_EQ(e0, en), placed before the plan's own predicates, within the same limit of
 * MZGPU_MFP_MAX_PREDICATES.  This is JoinClosure::apply: e0's error wins (it is evaluated first), a mismatch stops
 * evaluation before later expressions, and no map expression runs before them (their support is 0).
 *
 * Per match (key, va, vb) at time t and diff d (half join: the stream row's time and d1 * d2, wrapping; join_core:
 * max(t1, t2, meet)): at most one output row, the projection, once every predicate is TRUE and every map
 * expression has been evaluated without error; or one error row (code, payload, t, d), R32, in `errs`.  `out`
 * follows the rules of the bit-field closure entry points (probe order, consolidated when asked).  The half joins
 * append `errs` consolidated over the call; join_core appends them consolidated per slice, as it does its output.
 * The single-pass probe holds room for one error row per match, so no error row is ever dropped; with an MfpPlan
 * closure a half join takes that form within the same bytes as without one (an output and an error row per match).
 *
 * mzgpu_half_join_mfp[_buf] and mzgpu_half_join_many_mfp are mzgpu_half_join[_buf] and mzgpu_half_join_many with
 * the closure `jc` (jcs[j] for request j, none NULL); out rows are jc's out_row_bytes wide.  `errs` (R32) is not
 * any stream or output of the call.  mzgpu_join_new_mfp is mzgpu_join_new with `jc`; its work entry point is
 * mzgpu_join_core_work_mfp (deadline_ns as mzgpu_join_core_work_until, 0 = none), where fuel counts output and
 * error rows together (mz_join_core.rs:718-770); mzgpu_join_core_work[_until] on such a join is MZGPU_E_INVALID.
 * Out of scope: mzgpu_linear_join_new's plan, the fused initial closure of mzgpu_delta_first_stage_many and
 * mzgpu_update_stream (run mzgpu_mfp_step with a non-temporal plan, then mzgpu_half_join_many_mfp). */
typedef struct mzgpu_join_closure mzgpu_join_closure;
int32_t mzgpu_join_closure_new(mzgpu_ctx* ctx, const mzgpu_mfp* plan, const mzgpu_mfp_map* map,
                               mzgpu_join_closure** out);
void mzgpu_join_closure_free(mzgpu_join_closure* jc);
int32_t mzgpu_half_join_mfp(mzgpu_ctx* ctx, const mzgpu_r32* stream, uint64_t n, int32_t mem, mzgpu_spine* trace,
                            int32_t cmp_mode, const mzgpu_join_closure* jc, int32_t consolidate_output,
                            mzgpu_buf* out, mzgpu_buf* errs);
int32_t mzgpu_half_join_mfp_buf(mzgpu_ctx* ctx, mzgpu_buf* stream, mzgpu_spine* trace, int32_t cmp_mode,
                                const mzgpu_join_closure* jc, int32_t consolidate_output, mzgpu_buf* out,
                                mzgpu_buf* errs);
int32_t mzgpu_half_join_many_mfp(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf* const* streams, mzgpu_spine* const* traces,
                                 const int32_t* cmp_modes, const mzgpu_join_closure* const* jcs,
                                 mzgpu_buf* const* outs, mzgpu_buf* errs);
int32_t mzgpu_join_new_mfp(mzgpu_ctx* ctx, mzgpu_spine* trace1, mzgpu_spine* trace2, const mzgpu_join_closure* jc,
                           mzgpu_join** out);
int32_t mzgpu_join_core_work_mfp(mzgpu_join* j, uint64_t fuel_rows, uint64_t deadline_ns, mzgpu_buf* out,
                                 mzgpu_buf* errs, int32_t* done);

/* ---- FlatMap: a table function per input row, its rows appended to the input and run through the MfpPlan
 * (render_flat_map and drain_through_mfp, src/compute/src/render/flat_map.rs:29-200), for the table functions of
 * the fixed-width subset (TableFunc::eval, src/expr/src/relation/func.rs:3520-3620):
 *   MZGPU_TF_GENERATE_SERIES_INT32 / _INT64   args start, stop, step (INT32 programs / INT programs read as i64);
 *                        values start, start + step, ... while <= stop (step > 0) or >= stop (step < 0), stopping
 *                        on a checked-add overflow (num::range_step_inclusive, restated line for line by
 *                        TimestampRangeStepInclusive, func.rs:2884-2923).  The count is floor((stop - start) / step)
 *                        + 1 when the direction matches, else 0 (up to 2^64 rows for one input row); step == 0 is
 *                        InvalidParameterValue with payload 0.  One column: the value (int32 / int64).
 *   MZGPU_TF_GENERATE_SERIES_TIMESTAMP       args start, stop (TS programs); the step is the constant step_iv
 *                        (lo = microseconds as i64, hi = days in bits 0-31 | months in bits 32-63).  The same
 *                        series over i64 microseconds (generate_series_ts, func.rs:2925-2948); a zero step
 *                        (as_microseconds) is InvalidParameterValue with payload 0.  One column: the timestamp.
 *   MZGPU_TF_REPEAT_ROW                      arg n (INT): one row with diff n if n != 0 (func.rs:3283-3290).
 *   MZGPU_TF_REPEAT_ROW_NON_NEGATIVE         arg n (INT): n < 0 is InvalidParameterValue with payload n; 0 gives
 *                        nothing, otherwise one row with diff n (func.rs:3292-3306).
 *   MZGPU_TF_GUARD_SUBQUERY_SIZE             arg count (INT): 1 gives nothing, above 1 MultipleRowsFromSubquery,
 *                        below 0 NegativeRowsFromSubquery, 0 Internal (func.rs:3588-3606).  No rows, ever.
 * with_ordinality (WithOrdinality::eval, func.rs:3912-3960; allowed as TableFunc::with_ordinality allows it,
 * func.rs:3482-3517, so MZGPU_TF_REPEAT_ROW with it is MZGPU_E_INVALID): every function row with diff d >= 0
 * becomes d rows of diff 1, with an int64 ordinal from 1 as one more column.  So repeat_row_non_negative(n) with
 * ordinality yields n rows, with ordinals 1..n.
 *
 * The function's columns are extension columns 0, 1 of the row the MfpPlan sees: a program's MZGPU_HOP_COL /
 * COL_TS / COL_MZTS op or a projection field reads column i as source word MZGPU_SRC_FN0 + i (a series value as a
 * sign-extended i64 word, the ordinal as an i64).  An extension index at or beyond the function's column count
 * is MZGPU_E_INVALID.  The argument programs (n_ops[a] ops each, constants from `consts`, an interval in
 * MZGPU_HOP_TS_ADD_IV folded as in the MfpPlan) read the input row only: MZGPU_HOP_MAP and MZGPU_SRC_FN0 are
 * MZGPU_E_INVALID there.
 *
 * Per input row (words, time, diff), in order:
 *   1. the argument programs, in order; the first error becomes an error row at the input's (time, diff) and the
 *      row produces nothing more (flat_map.rs:75-85);
 *   2. the function; its error likewise becomes an error row at (time, diff);
 *   3. each function row (columns, d) is the row input ++ columns run through the MfpPlan exactly as
 *      mzgpu_mfp_new_map does (predicates, map expressions, temporal bounds, until, error rows, ready / held),
 *      at the input's time with diff d * diff, wrapping (flat_map.rs:168-199).
 * The new error codes follow MZGPU_MFP_ERR_TIMESTAMP_OUT_OF_RANGE.  They are raised by the function only and
 * never meet AND / OR, so their place in the numbering does not matter.
 *
 * An activation is mzgpu_flat_map_step[_buf] and then mzgpu_flat_map_work until *done.  The function rows of an
 * activation are numbered in input-row order, then series order; each call expands the next `fuel` of them
 * (fuel counts function rows before the MfpPlan; 0 is MZGPU_E_INVALID) and appends to `out`, consolidated, the
 * resulting updates with time < upper together with every held update that has become due, exactly as
 * mzgpu_mfp_step does; errors go to `errs`, consolidated.  `upper` belongs to the activation (the rules of
 * mzgpu_mfp_step apply).  What `out` and `errs` accumulate over an activation does not depend on `fuel`.  The
 * reference yields between input containers only (flat_map.rs:44-48, COMPUTE_FLAT_MAP_FUEL = 10^6,
 * src/compute-types/src/dyncfgs.rs:247-251); a device activation bounds each call's buffers by `fuel` instead.
 * The rows are copied when the activation starts, so the caller's buffer is free at once.  A step while an
 * activation is unfinished is MZGPU_E_FRONTIER and changes nothing; work with no activation pending is a no-op
 * that sets *done.  A step waits for the device once (for the 128-bit count of the activation's function rows,
 * counted in mzgpu_stats.host_syncs); work never waits for its own sake.
 *
 * mzgpu_flat_map_frontier(op, &t): the least held time or, while an activation is unfinished, the least input
 * time among the rows not yet fully expanded if that is lower; MZGPU_FRONTIER_EMPTY if neither exists.
 * mzgpu_flat_map_stats(op, out): out[0..2] as mzgpu_mfp_stats, out[3] = function rows still to expand in the
 * activation (saturating at u64::MAX).  Both wait for the device.
 *
 * Refused on the host, leaving no operator and the context usable: MZGPU_E_INVALID for a wrong argument count or
 * argument types, MZGPU_HOP_MAP in an argument program, an extension column at or beyond the function's column
 * count, MZGPU_TF_REPEAT_ROW with ordinality, and everything mzgpu_mfp_new_map refuses as invalid;
 * MZGPU_E_UNSUPPORTED for a timestamp step with months or beyond i64 microseconds, any other table function
 * (JSON, arrays, lists, maps, regexes, CSV, Wrap, timestamptz series, ROWS FROM) and everything mzgpu_mfp_new_map
 * refuses as unsupported. */
#define MZGPU_TF_GENERATE_SERIES_INT32 1
#define MZGPU_TF_GENERATE_SERIES_INT64 2
#define MZGPU_TF_GENERATE_SERIES_TIMESTAMP 3
#define MZGPU_TF_REPEAT_ROW 4
#define MZGPU_TF_REPEAT_ROW_NON_NEGATIVE 5
#define MZGPU_TF_GUARD_SUBQUERY_SIZE 6
#define MZGPU_SRC_FN0 8 /* mzgpu_field.src / MZGPU_HOP_COL* arg of extension column 0 */
#define MZGPU_SRC_FN(i) (MZGPU_SRC_FN0 + (i))
#define MZGPU_TF_ERR_INVALID_PARAMETER_VALUE 8
#define MZGPU_TF_ERR_MULTIPLE_ROWS_FROM_SUBQUERY 9
#define MZGPU_TF_ERR_NEGATIVE_ROWS_FROM_SUBQUERY 10
#define MZGPU_TF_ERR_INTERNAL 11
typedef struct mzgpu_table_func {
  uint32_t kind; /* MZGPU_TF_* */
  uint32_t with_ordinality;
  uint32_t n_consts;
  uint32_t n_ops[3]; /* argument programs; unused arguments have 0 ops */
  mzgpu_having_op ops[3][MZGPU_MFP_MAX_OPS];
  mzgpu_having_const consts[MZGPU_MFP_MAX_CONSTS];
  mzgpu_having_const step_iv; /* MZGPU_TF_GENERATE_SERIES_TIMESTAMP: the step interval */
} mzgpu_table_func;
typedef struct mzgpu_flat_map_op mzgpu_flat_map_op;
int32_t mzgpu_flat_map_new(mzgpu_ctx* ctx, const mzgpu_table_func* func, const mzgpu_mfp* plan,
                           const mzgpu_mfp_map* map, uint64_t until, mzgpu_flat_map_op** out);
void mzgpu_flat_map_free(mzgpu_flat_map_op* op);
int32_t mzgpu_flat_map_step(mzgpu_flat_map_op* op, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                            uint64_t fuel, mzgpu_buf* out, mzgpu_buf* errs, int32_t* done);
int32_t mzgpu_flat_map_step_buf(mzgpu_flat_map_op* op, mzgpu_buf* rows, uint64_t upper, uint64_t fuel,
                                mzgpu_buf* out, mzgpu_buf* errs, int32_t* done);
int32_t mzgpu_flat_map_work(mzgpu_flat_map_op* op, uint64_t fuel, mzgpu_buf* out, mzgpu_buf* errs, int32_t* done);
int32_t mzgpu_flat_map_frontier(mzgpu_flat_map_op* op, uint64_t* out);
int32_t mzgpu_flat_map_stats(mzgpu_flat_map_op* op, uint64_t out[4]);

/* ------------------------------ f1 (first step): Row keys as fixed-width words */
/* A `Row` orders by byte length first, then by its bytes (RowRef::cmp,
 * src/repr/src/row.rs:704-722; the arrangement key order of RowRowSpine,
 * src/compute/src/row_spine.rs:116-290).  A Row of at most 7 bytes maps to one u64 that
 * orders the same way and maps back: key = len << 56 | bytes, big-endian, zero padded.
 * (Materialize encodes small integers in 2-5 bytes, src/repr/src/row.rs: the tag byte plus a
 * minimal-width payload, so single-column integer keys usually fit.)  Pure host functions:
 * no context, no device.  MZGPU_E_UNSUPPORTED for longer rows: such an arrangement stays on
 * the Rust path until variable-width keys are built (SURVEY 8f-1). */
int32_t mzgpu_rowkey_pack(const uint8_t* row_bytes, uint64_t len, uint64_t* key_out);
/* n rows stored back to back, row i = data[offsets[i] .. offsets[i + 1]) (the layout of a
 * columnar Row container).  Stops at the first row that does not fit: returns
 * MZGPU_E_UNSUPPORTED and *n_done = rows packed. */
int32_t mzgpu_rowkeys_pack(const uint8_t* data, const uint64_t* offsets, uint64_t n, uint64_t* keys_out,
                           uint64_t* n_done);
/* Inverse: writes `len` bytes (at most 7) to row_bytes_out. */
int32_t mzgpu_rowkey_unpack(uint64_t key, uint8_t row_bytes_out[7], uint64_t* len_out);

/* --------------------------------------- row L: linear join plans */
/* LinearJoinPlan (src/compute-types/src/plan/join/linear_join.rs:26-62) as rendered by
 * LinearJoinSpec::render / differential_join (src/compute/src/render/join/linear_join.rs:230-527):
 * the running result starts as the source relation, and every stage (a) re-keys it by the stage's
 * stream_key, keeping the thinned columns as the value ("LinearJoinKeyPreparation", :343-383),
 * (b) arranges it ("JoinStage": Batcher -> seal -> Spine, :387-398) and (c) joins the arrangement
 * with the stage's lookup arrangement through mz_join_core with the stage's JoinClosure
 * (differential_join_inner, :462-527); initial / final closures are per-row maps in front of the
 * first stage and behind the last one (:243-266, :296-316).  Closures are POD descriptors as
 * everywhere on this boundary; the key preparation of a stage is one too (key fields = stream_key,
 * val fields = stream_thinning, evaluated on the running (key, val) row with val2 = 0). */
#define MZGPU_LINEAR_MAX_STAGES 6
typedef struct mzgpu_linear_stage_plan {
  mzgpu_closure stream_key; /* (key, val) of the running result -> (stage key, thinned val) */
  mzgpu_closure closure;    /* JoinClosure on (key, stream val, lookup val) -> next running row */
} mzgpu_linear_stage_plan;
typedef struct mzgpu_linear_join_plan {
  int32_t has_initial_closure; /* 0: identity */
  int32_t has_final_closure;   /* 0: identity */
  uint32_t n_stages;           /* 1 .. MZGPU_LINEAR_MAX_STAGES */
  uint32_t _pad;
  mzgpu_closure initial_closure;
  mzgpu_closure final_closure;
  mzgpu_linear_stage_plan stages[MZGPU_LINEAR_MAX_STAGES];
} mzgpu_linear_join_plan;
typedef struct mzgpu_linear_join mzgpu_linear_join;
/* lookup_traces[s] = the arrangement of stage s's lookup relation by its lookup_key (owned by the
 * caller, who inserts the relation's batches and advances its compaction); the operator owns the
 * "JoinStage" arrangements of the running result.  A plan the descriptors cannot express is
 * MZGPU_E_UNSUPPORTED / MZGPU_E_INVALID here, at render time. */
int32_t mzgpu_linear_join_new(mzgpu_ctx* ctx, const mzgpu_linear_join_plan* plan, mzgpu_spine* const* lookup_traces,
                              mzgpu_linear_join** out);
void mzgpu_linear_join_free(mzgpu_linear_join* lj);
/* One activation: the frontier advances to `upper` (every update of this activation is at a time
 * in [previous upper, upper)).  `source` = the source relation's new updates (R32, may be empty or
 * NULL), lookup_batches[s] = the batch the caller has just inserted into lookup_traces[s] (NULL: that
 * relation did not change).  The final collection's new updates are APPENDED to `out` (R32).  Stage
 * by stage: key preparation, seal of the stage arrangement at `upper`, join_core over the new batches
 * of both sides (fuel: to completion), result handed to the next stage -- no row count returns to
 * the host in between beyond what join_core itself reads. */
int32_t mzgpu_linear_join_step(mzgpu_linear_join* lj, mzgpu_buf* source, mzgpu_batch* const* lookup_batches,
                               uint64_t upper, mzgpu_buf* out);
/* The "JoinStage" arrangement of stage s (logical compaction is the caller's call, as for any
 * arrangement; physical compaction follows the acknowledged frontiers inside the operator). */
mzgpu_spine* mzgpu_linear_join_stage_trace(mzgpu_linear_join* lj, uint32_t stage);

/* ------------------------------------ f4: the columnar wire format */
/* `Column<C>` (src/timely-util/src/columnar.rs:54-222) is the container the reference moves
 * update batches in: between workers (`ContainerBytes::{from_bytes, into_bytes}`, :177-222), out
 * of `ColumnBuilder` (src/timely-util/src/columnar/builder.rs:28-111) and into the merge batcher
 * (`Col2ValBatcher`, columnar.rs:41-45).  Serialized (`Column::Bytes` / `Column::Align`) it is
 * `columnar::bytes::indexed` (crate columnar 0.12.1, not vendored; layout pinned by the
 * reference's `raw_columnar_bytes`, columnar.rs:247-258): word 0 = 8 * (k + 1), words 1..k = the
 * byte offset where each of the k slices ends (a slice starts at the previous end rounded up to 8),
 * then the slices, zero padded to whole words.  These entry points move between that format and
 * the row buffers of this library ON THE DEVICE (one transposing kernel each way), so that a
 * worker can hand over the bytes it received or ship the bytes it must send without a host-side
 * row loop:
 *   MZGPU_COLUMN_U64X4   Column<((u64, u64), u64, i64)>: 4 slices key, val, time, diff <-> R32
 *   MZGPU_COLUMN_U64X2   Column<(u64, i64)>: 2 slices key, diff                       <-> R16
 *   MZGPU_COLUMN_ROWROW  Column<((Row, Row), Timestamp, Diff)>: 6 slices key bounds (the END
 *                        offset of every row, src/repr/src/row.rs:447-452,606-611), key bytes,
 *                        val bounds, val bytes, times, diffs <-> R32 whose key and val are Rows
 *                        of at most 7 bytes packed as by mzgpu_rowkey_pack (a longer Row:
 *                        MZGPU_E_UNSUPPORTED, nothing appended) */
#define MZGPU_COLUMN_U64X4 0
#define MZGPU_COLUMN_U64X2 1
#define MZGPU_COLUMN_ROWROW 2
/* indexed::length_in_words of a container of `rows` updates; key_bytes / val_bytes = total Row
 * bytes (ROWROW only, else ignored).  Pure host function. */
uint64_t mzgpu_column_length_in_words(int32_t layout, uint64_t rows, uint64_t key_bytes, uint64_t val_bytes);
/* The ship signal shared by ColumnBuilder::push_into (builder.rs:48-52) and
 * `at_serialized_capacity` (columnar.rs:164-175): 1 when `words` is within 10 % of the next
 * multiple of 2 MiB (2^18 words).  Pure host function. */
int32_t mzgpu_column_at_capacity(uint64_t words);
/* Rows of the container ColumnBuilder mints for a fixed-width layout (the smallest row count at
 * which the ship signal fires); 0 for ROWROW, where it depends on the data. */
uint64_t mzgpu_column_ship_rows(int32_t layout);
/* `Column::borrow()` + drain: APPEND the updates of one serialized container (`n_words` words in
 * host or device memory, 8-byte aligned as `Column::Align` guarantees) to `out` (R32, or R16 for
 * U64X2).  The index is validated on the host (MZGPU_E_INVALID: not a container of this layout;
 * for device memory the k + 1 index words are read back first).  ROWROW waits for the device once
 * (bounds are validated and over-long Rows detected there). */
int32_t mzgpu_column_decode(mzgpu_ctx* ctx, int32_t layout, const uint64_t* words, uint64_t n_words, int32_t mem,
                            mzgpu_buf* out);
/* `indexed::encode` of rows [first, first + n) of `rows` (clamped to its length) into `words`
 * (host or device memory, capacity cap_words); *n_words = words written.  MZGPU_E_CAPACITY with
 * *n_words = the size needed if cap_words is too small.  Waits for the device (the caller needs
 * the size to ship the bytes). */
int32_t mzgpu_column_encode(mzgpu_buf* rows, int32_t layout, uint64_t first, uint64_t n, uint64_t* words,
                            uint64_t cap_words, int32_t mem, uint64_t* n_words);
/* ColumnBuilder over a whole buffer: the containers push_into would mint for these rows in order,
 * then the remainder (`finish`), written back to back into `words`; chunk_words[i] = size of
 * container i, *n_chunks = their number.  MZGPU_E_CAPACITY (with the totals needed in *n_words
 * and *n_chunks) if either capacity is too small. */
int32_t mzgpu_column_build(mzgpu_buf* rows, int32_t layout, uint64_t* words, uint64_t cap_words, int32_t mem,
                           uint64_t* n_words, uint64_t* chunk_words, uint32_t cap_chunks, uint32_t* n_chunks);
/* walk_cursor over one batch into a container (src/compute/src/render/context.rs:1299-1355; the
 * read side of an arrangement import / peek): rows [first, first + fuel) of the batch in cursor
 * order -- a sealed batch is consolidated, so the per-(key, val) consolidation of the walk is the
 * identity -- encoded as by mzgpu_column_encode.  With `key` non-NULL only that key's rows are
 * walked (seek_key); *n_rows = rows emitted (the caller resumes at first + *n_rows while it equals
 * fuel). */
int32_t mzgpu_batch_walk_column(mzgpu_batch* batch, const uint64_t* key, uint64_t first, uint64_t fuel,
                                int32_t layout, uint64_t* words, uint64_t cap_words, int32_t mem,
                                uint64_t* n_words, uint64_t* n_rows);

/* --------------------------------- f3: the MV sink's correction buffer */
/* CorrectionV2 (src/compute/src/sink/correction_v2.rs:213-498): the difference between the
 * desired and the persisted contents of a materialized view, as R32 updates
 * ((key, val), time, diff).  insert / insert_negated add (negated) updates, with times
 * advanced to `since`; updates_before(upper) appends to `out` every update whose advanced
 * time is before `upper`, consolidated and ordered by (time, key, val) (nothing if
 * !(since < upper)); advance_since moves `since` forward (MZGPU_FRONTIER_EMPTY discards
 * everything); consolidate_at_since compacts the updates at `since`.  The reference's chains
 * of chunks are an amortisation device of the CPU implementation: here inserts are stashed
 * and a read consolidates everything buffered in one pass (same results). */
typedef struct mzgpu_correction mzgpu_correction;
int32_t mzgpu_correction_new(mzgpu_ctx* ctx, mzgpu_correction** out);
void mzgpu_correction_free(mzgpu_correction* c);
int32_t mzgpu_correction_insert(mzgpu_correction* c, const mzgpu_r32* rows, uint64_t n, int32_t mem, int32_t negate);
int32_t mzgpu_correction_insert_buf(mzgpu_correction* c, mzgpu_buf* rows, int32_t negate);
int32_t mzgpu_correction_updates_before(mzgpu_correction* c, uint64_t upper, mzgpu_buf* out);
int32_t mzgpu_correction_advance_since(mzgpu_correction* c, uint64_t since);
int32_t mzgpu_correction_consolidate_at_since(mzgpu_correction* c);
/* Updates held (after consolidating what is buffered; waits for the device). */
uint64_t mzgpu_correction_len(mzgpu_correction* c);

/* ------------------------------------------------------- a13: exchange */
/* Bytes of the NCCL unique id passed to mzgpu_comm_init. */
#define MZGPU_COMM_ID_BYTES 128
/* Rank 0 creates the id; the host distributes it (timely's own bootstrap,
 * src/cluster/src/communication.rs:288, stays on the host). */
int32_t mzgpu_comm_unique_id(uint8_t id[MZGPU_COMM_ID_BYTES]);
int32_t mzgpu_comm_init(mzgpu_ctx* ctx, const uint8_t id[MZGPU_COMM_ID_BYTES]);
/* Exchange pact by key hash (src/compute/src/extensions/arrange.rs:116,
 * src/timely-util/src/columnar.rs:227-237): route each row to
 * hash(key) % peers; collective over all peers' contexts (all must call in the
 * same order).  `in` and `out` are R32 or RACC buffers; `out` is replaced. */
int32_t mzgpu_exchange(mzgpu_ctx* ctx, mzgpu_buf* in, mzgpu_buf* out);
/* k independent exchanges in one round (one counts all-to-all, one host wait, one
 * payload all-to-all): the exchange points of operators that run side by side,
 * e.g. the arrangement inputs of one timestamp.  k <= 8; all peers pass the same k. */
int32_t mzgpu_exchange_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** ins, mzgpu_buf** outs);
/* ---- the same pact over peer memory (NVLink / NVSwitch): no NCCL, no host wait.
 * Every worker owns a landing zone with a fixed-capacity region per (buffer slot, source
 * worker); an exchange round is ONE scatter kernel that partitions the rows and writes them
 * straight into the destination workers' zones (peer stores), publishing counts and a round
 * flag, and ONE gather kernel that waits for all sources' flags on the device and compacts
 * the regions into the operator's input buffer, leaving the row count on the device.
 * Setup (once, host bootstrap as for mzgpu_comm_init): every worker calls _export, the 64-byte
 * handles are all-gathered by the host, every worker calls _import with all of them (index =
 * worker).  `landing_rows` = capacity of one region: no worker may send more than that many
 * rows of one buffer to one destination in one round (violations are detected on the device
 * and reported as MZGPU_E_CAPACITY at the next read-back; nothing wrong is delivered);
 * `region_row_bytes` = widest row exchanged (32 or 80).  Zone size = 4 KB + 2 x 8 x peers x
 * landing_rows x region_row_bytes bytes. */
#define MZGPU_P2P_HANDLE_BYTES 64
int32_t mzgpu_comm_p2p_export(mzgpu_ctx* ctx, uint64_t landing_rows, uint32_t region_row_bytes,
                              uint8_t handle[MZGPU_P2P_HANDLE_BYTES]);
int32_t mzgpu_comm_p2p_import(mzgpu_ctx* ctx, const uint8_t* handles /* peers x 64 bytes */);
/* Same-process variant (several workers of one process, e.g. one thread per GPU, or a test
 * that runs every worker on one GPU): zones[w] = worker w's mzgpu_comm_p2p_zone(). */
void* mzgpu_comm_p2p_zone(mzgpu_ctx* ctx);
int32_t mzgpu_comm_p2p_import_local(mzgpu_ctx* ctx, void* const* zones);
/* One round for k buffers (all workers call with the same k, in the same order).
 * outs[e] is replaced; its capacity is recv_ub[e] rows if given (the caller's bound on what
 * this worker can receive, e.g. the global batch size), else peers x landing_rows.
 * mzgpu_exchange_p2p = _send (scatter) followed by _recv (gather). */
int32_t mzgpu_exchange_p2p(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** ins, mzgpu_buf** outs, const uint64_t* recv_ub);
int32_t mzgpu_exchange_p2p_send(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** ins);
int32_t mzgpu_exchange_p2p_recv(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** outs, const uint64_t* recv_ub);
/* The routing function itself (for tests and host-side pre-partitioning). */
uint32_t mzgpu_route(uint64_t key, uint32_t peers);
/* ---- index peeks: a SELECT against an arrangement at a timestamp (IndexPeek::seek_fulfillment and
 * collect_finished_data, src/compute/src/compute_state.rs:1433-1673; PeekResultIterator,
 * src/compute/src/compute_state/peek_result_iterator.rs:40-304; RowSetFinishing, src/expr/src/relation.rs:3526-3646).
 *
 * The ok trace is an R32 (key, val) arrangement (mzgpu_spine of 32-byte rows); the optional error trace holds R32
 * rows (code, payload, time, diff), the error rows every operator here emits, arranged by the caller.
 *
 * mzgpu_peek_plan_new(ctx, plan, map, fin, out) checks the plan once with the validation of mzgpu_mfp_new_map and
 * keeps it, with the finishing, in device memory.  plan->in_row_bytes is 32 (the rows (key, val) the trace holds,
 * MZGPU_SRC_KEY / VAL1); out_row_bytes is 32 or 40.  Refused, leaving no handle and the context usable:
 * in_row_bytes != 32 and n_temporal != 0 (a peek's plan is a SafeMfpPlan: the adapter has replaced mz_now() by the
 * timestamp) with MZGPU_E_INVALID, everything mzgpu_mfp_new_map refuses with its status, and a malformed finishing
 * (more than MZGPU_MAX_ORDER_LANES lanes, unknown lane flags, a field outside the output row) with MZGPU_E_INVALID;
 * a float64 order lane and a negative limit with MZGPU_E_UNSUPPORTED.  fin == NULL is no ORDER BY, no LIMIT, no
 * OFFSET and the identity projection.  A call using the handle must not outlive it.
 *
 * mzgpu_finishing: order lanes read the plan's OUTPUT words (field.src MZGPU_SRC_KEY / VAL1 / VAL2 are output words 0,
 * 1 and 2), encoded as the TopK rows are (signed lanes ^ 2^63, descending lanes complemented); limit (MZGPU_TOPK_NO_LIMIT
 * = none), offset; and the projection, per output word an OR of bit-fields of the output words (as mzgpu_mfp's
 * fields; no field for any word = the identity).  Order lanes may read words the projection then drops.
 *
 * mzgpu_peek_many(ctx, ok, errs_or_NULL, k, reqs, outs, results): k requests (1..MZGPU_PEEK_MANY_MAX), each with its
 * plan, as_of, literal keys and max_rows.  literals == NULL is a full scan; otherwise the n_literals keys (in
 * literals_mem space) are looked up, a duplicate once, so n_literals == 0 finds no rows.  For request i, results[i]:
 *   MZGPU_PEEK_NOT_READY  the upper of the ok trace or of the error trace is <= as_of (nothing is appended);
 *   MZGPU_PEEK_ERROR      kind and detail words, in this precedence:
 *     MZGPU_PEEK_ERR_SINCE            the logical compaction of either trace is beyond as_of: (since, as_of)
 *     MZGPU_PEEK_ERR_ERRS_ROW         the first (code, payload), in cursor order, of the error trace whose count at
 *                                     as_of is positive: (code, payload)
 *     MZGPU_PEEK_ERR_ERRS_RETRACTION  that first non-zero count is negative: (code, payload, count)
 *     MZGPU_PEEK_ERR_MFP              the first failure in (key, val) order is an MfpPlan error: (code, payload, key, val)
 *     MZGPU_PEEK_ERR_RETRACTION       ... a pair the plan keeps with a negative count: (key, val, count)
 *     MZGPU_PEEK_ERR_TOO_LARGE        the finishing keeps more than max_rows rows (0 = no limit): (rows)
 *   MZGPU_PEEK_ROWS       n_rows rows appended to outs[i] (the plan's out_row_bytes wide): (w0, w1[, w2], as_of,
 *                         copies) in finishing order, copies clipped by the [offset, offset + limit) cut.
 * Per pair (key, val) with time <= as_of accumulated to a non-zero count, in (key, val) order: the plan runs; an error
 * fails the peek, a filtered pair is skipped (its count is never checked), a kept pair with a negative count fails it,
 * and a kept pair gives its output row with the count as copies.  Output rows equal before the projection are one
 * row (their copies summed); rows that become equal through the projection are not merged.
 *
 * Fixed-width stand-ins, chosen deliberately:
 *   1. pairs with no count at as_of are not evaluated (the reference also runs the plan on pairs still physically in
 *      the trace with a zero sum or only future times, which makes its errors depend on compaction state);
 *   2. rows equal on every order lane are ordered by the output row's words as unsigned (before the projection), as
 *      the TopK operators document;
 *   3. LIMIT without ORDER BY keeps the first rows in that word order (the reference takes them in cursor order;
 *      SQL allows any bag);
 *   4. max_rows counts the rows the finishing keeps, in place of max_result_size's bytes of variable-width rows;
 *   5. the literal columns an IndexedFilter appends equal the key by construction: the caller lowers them to
 *      MZGPU_SRC_KEY.
 *
 * No peek modifies a trace: no compaction, no merge work, batches are only read (batches still being built through
 * their device headers, a merge in flight on the side stream through its inputs).  A trace of more than 64 non-empty
 * batches is MZGPU_E_UNSUPPORTED, as for the probes.  The call waits for the device once, for all k requests, to read
 * the results: the answer goes to a client.  It waits before that only where the probes and the consolidation do: a
 * call with literal requests first reads the row counts of the ok trace's batches still being built (the probe's
 * fan-out bound needs them), a lookup on key runs longer than 1,024 rows counts its matches first, and more than
 * 32 Mi gathered rows have their count read back before they are consolidated.  Device memory: the full scans are
 * gathered once per distinct as_of, (ok trace rows) x (distinct as_of of the full scans) + (error trace rows) x
 * (distinct as_of) rows of 40 bytes; the finishing rows, 72 bytes each, are at most one per kept pair and request
 * at that pair's as_of.  mzgpu_peek is mzgpu_peek_many with k = 1.  A refused call (MZGPU_E_INVALID /
 * _UNSUPPORTED) appends nothing and leaves results unspecified. */
#define MZGPU_PEEK_MANY_MAX 64
#define MZGPU_PEEK_ROWS 0
#define MZGPU_PEEK_NOT_READY 1
#define MZGPU_PEEK_ERROR 2
#define MZGPU_PEEK_ERR_SINCE 1
#define MZGPU_PEEK_ERR_ERRS_ROW 2
#define MZGPU_PEEK_ERR_ERRS_RETRACTION 3
#define MZGPU_PEEK_ERR_MFP 4
#define MZGPU_PEEK_ERR_RETRACTION 5
#define MZGPU_PEEK_ERR_TOO_LARGE 6
typedef struct mzgpu_finishing {
  uint32_t n_order;
  mzgpu_order_lane order[MZGPU_MAX_ORDER_LANES];
  int64_t limit;   /* MZGPU_TOPK_NO_LIMIT = none */
  uint64_t offset;
  uint32_t n_project[3]; /* fields of projected word 0, 1, 2 (2: 40-byte output only); all 0 = identity */
  mzgpu_field project[3][MZGPU_MAX_FIELDS];
} mzgpu_finishing;
typedef struct mzgpu_peek_plan mzgpu_peek_plan;
typedef struct mzgpu_peek_req {
  const mzgpu_peek_plan* plan;
  uint64_t as_of;
  const uint64_t* literals; /* NULL = full scan */
  uint64_t n_literals;
  int32_t literals_mem;     /* MZGPU_MEM_HOST / MZGPU_MEM_DEVICE */
  uint64_t max_rows;        /* 0 = none */
} mzgpu_peek_req;
typedef struct mzgpu_peek_result {
  int32_t status;   /* MZGPU_PEEK_ROWS / NOT_READY / ERROR */
  int32_t err_kind; /* MZGPU_PEEK_ERR_* for MZGPU_PEEK_ERROR, else 0 */
  uint64_t n_rows;  /* rows appended to the request's output */
  uint64_t detail[4];
} mzgpu_peek_result;
int32_t mzgpu_peek_plan_new(mzgpu_ctx* ctx, const mzgpu_mfp* plan, const mzgpu_mfp_map* map, const mzgpu_finishing* fin,
                            mzgpu_peek_plan** out);
void mzgpu_peek_plan_free(mzgpu_peek_plan* p);
int32_t mzgpu_peek_many(mzgpu_ctx* ctx, mzgpu_spine* ok, mzgpu_spine* errs, uint32_t k, const mzgpu_peek_req* reqs,
                        mzgpu_buf* const* outs, mzgpu_peek_result* results);
int32_t mzgpu_peek(mzgpu_ctx* ctx, mzgpu_spine* ok, mzgpu_spine* errs, const mzgpu_peek_req* req, mzgpu_buf* out,
                   mzgpu_peek_result* result);

/* The device half of an exchange round on its own: the k buffers are bucketed by
 * destination for `peers` workers (any 1 <= peers <= 64, independent of the ctx's
 * own peer count) with the kernels mzgpu_exchange_many runs; outs[e] receives the
 * rows of ins[e] grouped by destination in worker order, counts[e * peers + p] the
 * rows bound for worker p (read back: one host wait).  Row order inside a
 * destination group is unspecified (the receiving Batcher sorts).  Lets a host
 * that moves the bytes itself (timely's own network layer) keep the partitioning
 * on the GPU, and lets one GPU test the routing for any cluster size. */
int32_t mzgpu_partition_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** ins, uint32_t peers, mzgpu_buf** outs,
                             uint64_t* counts);

#ifdef __cplusplus
}
#endif
#endif /* MZGPU_H */
