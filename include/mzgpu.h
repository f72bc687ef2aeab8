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
 * operator evaluates a key's values directly and reports MZGPU_E_UNSUPPORTED (at the next
 * read-back) for a key with more than 32 distinct live values. */
#define MZGPU_AGG_MIN 4
#define MZGPU_AGG_MAX 5
/* TopK per key (BasicTopKPlan, src/compute/src/render/top_k.rs:215-248 and the reduction logic of
 * build_topk_negated_stage, :521-673): over the key's live (value, count) pairs -- any non-positive
 * count yields the error row (flags bit1, diff 1); otherwise the values are ordered (ascending, or
 * descending), `offset` rows are skipped and at most `limit` rows kept, counting multiplicities.
 * The operator emits the changes of that window directly (the reference emits its negated complement
 * and concatenates it with the input: the same collection).  ROUT rows: sum_lo = the value,
 * diff = the change of the value's multiplicity inside the window, count = sum_hi = 0.  The staged
 * bucket tree (build_topk, :251-380) bounds per-key work for huge groups; as for MIN/MAX a key with more
 * than 32 distinct live values is reported MZGPU_E_UNSUPPORTED.  Created by mzgpu_topk_new. */
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
 * R32 (KeyValBatcher) or RACC (the accumulable arrangement's batcher). */
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
