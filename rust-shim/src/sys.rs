//! FFI declarations for libmzgpu.so (include/mzgpu.h).  UNCOMPILED: see ../README.md.
#![allow(non_camel_case_types, dead_code)]
use std::os::raw::{c_char, c_void};

#[repr(C)] #[derive(Clone, Copy, Debug, Default, PartialEq, Eq, PartialOrd, Ord)]
pub struct R32 { pub key: u64, pub val: u64, pub time: u64, pub diff: i64 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)]
pub struct Desc { pub lower: u64, pub upper: u64, pub since: u64 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)]
pub struct KeyRun { pub key: u64, pub first: u64, pub len: u64 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)]
pub struct ArrangementSize { pub size_bytes: u64, pub capacity_bytes: u64, pub allocations: u64, pub batches: u64, pub updates: u64 }
#[repr(C)] pub struct Closure { _b: [u8; 144] }
#[repr(C)] #[derive(Clone, Copy, Debug, Default, PartialEq, Eq, PartialOrd, Ord)]
pub struct R16 { pub key: u64, pub diff: i64 }
/// Output correction of the reduce operators (mzgpu_rout, 64 bytes).
#[repr(C)] #[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub struct Rout { pub key: u64, pub count: i64, pub sum_lo: u64, pub sum_hi: i64, pub flags: u64, pub time: u64, pub diff: i64, pub _pad: i64 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)]
pub struct Stats {
    pub kernel_launches: u64, pub device_bytes_in_use: u64, pub device_bytes_peak: u64, pub rows_in: u64,
    pub rows_out: u64, pub h2d_bytes: u64, pub d2h_bytes: u64, pub host_syncs: u64,
}

pub enum Ctx {} pub enum Buf {} pub enum Batcher {} pub enum Builder {} pub enum Batch {}
pub enum Spine {} pub enum Join {} pub enum Reduce {} pub enum Correction {}

pub const OK: i32 = 0;
pub const E_INVALID: i32 = -1;
pub const E_CUDA: i32 = -2;
pub const E_CAPACITY: i32 = -3;
pub const E_UNSUPPORTED: i32 = -4;
pub const E_NCCL: i32 = -5;
pub const E_FRONTIER: i32 = -6;
pub const MEM_HOST: i32 = 0;
pub const MEM_DEVICE: i32 = 1;
pub const FRONTIER_EMPTY: u64 = u64::MAX;
pub const ROW_R32: u32 = 32;
pub const ROW_RACC: u32 = 80;
pub const ROW_ROUT: u32 = 64;
pub const HALFJOIN_LE: i32 = 0;
pub const HALFJOIN_LT: i32 = 1;
pub const AGG_COUNT_SUM_I64: i32 = 0;
pub const AGG_COUNT_SUM_F64: i32 = 1;
pub const AGG_DISTINCT: i32 = 2;
pub const AGG_THRESHOLD: i32 = 3;
pub const AGG_MIN: i32 = 4;
pub const AGG_MAX: i32 = 5;
pub const AGG_TOPK: i32 = 6;
pub const MAX_ACCUM_LANES: usize = 8;
/// OR'd into `AccumLane::kind`: the lane is COUNT(DISTINCT col) / SUM(DISTINCT col) (int64 lanes only).
pub const ACCUM_DISTINCT: i32 = 0x100;
/// A column pick (mzgpu_field): bits [shift, shift + bits) of word `src`.
#[repr(C)] #[derive(Clone, Copy, Debug, Default)]
pub struct Field { pub src: u8, pub shift: u8, pub bits: u8, pub dst_shift: u8 }
/// One aggregate lane of the multi-column accumulable reduce (mzgpu_accum_lane).
#[repr(C)] #[derive(Clone, Copy, Debug, Default)]
pub struct AccumLane { pub kind: i32, pub sign_extend: u32, pub field: Field }
pub const COMM_ID_BYTES: usize = 128;
pub const P2P_HANDLE_BYTES: usize = 64;

#[link(name = "mzgpu")]
extern "C" {
    pub fn mzgpu_ctx_create(device: i32, worker_index: i32, peers: i32, out: *mut *mut Ctx) -> i32;
    pub fn mzgpu_ctx_destroy(ctx: *mut Ctx);
    pub fn mzgpu_ctx_sync(ctx: *mut Ctx) -> i32;
    pub fn mzgpu_last_error(ctx: *mut Ctx) -> *const c_char;
    // a2-a4: batcher
    pub fn mzgpu_batcher_new(ctx: *mut Ctx, row_bytes: u32, out: *mut *mut Batcher) -> i32;
    pub fn mzgpu_batcher_free(b: *mut Batcher);
    pub fn mzgpu_batcher_push(b: *mut Batcher, rows: *const c_void, n: u64, mem: i32) -> i32;
    pub fn mzgpu_batcher_seal(b: *mut Batcher, upper: u64, batch: *mut *mut Batch, new_lower: *mut u64) -> i32;
    pub fn mzgpu_batcher_frontier(b: *mut Batcher) -> u64;
    // a5: builder, batches
    pub fn mzgpu_builder_new(ctx: *mut Ctx, row_bytes: u32, capacity_rows: u64, out: *mut *mut Builder) -> i32;
    pub fn mzgpu_builder_free(b: *mut Builder);
    pub fn mzgpu_builder_push(b: *mut Builder, rows: *const c_void, n: u64, mem: i32) -> i32;
    pub fn mzgpu_builder_done(b: *mut Builder, desc: Desc, out: *mut *mut Batch) -> i32;
    pub fn mzgpu_batch_len(b: *const Batch) -> u64;
    pub fn mzgpu_batch_keys(b: *const Batch) -> u64;
    pub fn mzgpu_batch_desc(b: *const Batch) -> Desc;
    pub fn mzgpu_batch_retain(b: *mut Batch);
    pub fn mzgpu_batch_release(b: *mut Batch);
    pub fn mzgpu_batch_merge(b1: *mut Batch, b2: *mut Batch, since: u64, out: *mut *mut Batch) -> i32;
    // a8: cursors (batched)
    pub fn mzgpu_batch_seek_keys(b: *mut Batch, keys: *const u64, n: u64, mem: i32, runs: *mut KeyRun) -> i32;
    pub fn mzgpu_batch_key_page(b: *mut Batch, first_ordinal: u64, max_keys: u64, mem: i32, runs: *mut KeyRun, n_out: *mut u64) -> i32;
    pub fn mzgpu_batch_rows(b: *mut Batch, first: u64, len: u64, rows: *mut c_void, mem: i32) -> i32;
    pub fn mzgpu_batch_index_export(b: *mut Batch, slots: *mut c_void, cap_slots: u64, mem: i32, n_slots: *mut u64,
                                    n_keys: *mut u64, longest_run: *mut u64) -> i32;
    // a6, a14: spine
    pub fn mzgpu_spine_new(ctx: *mut Ctx, row_bytes: u32, effort: u32, out: *mut *mut Spine) -> i32;
    pub fn mzgpu_spine_free(s: *mut Spine);
    pub fn mzgpu_spine_insert(s: *mut Spine, batch: *mut Batch) -> i32;
    pub fn mzgpu_spine_exert(s: *mut Spine, effort: u64, did_work: *mut i32) -> i32;
    pub fn mzgpu_spine_exert_logic(s: *const Spine, proportionality: u32) -> u64;
    pub fn mzgpu_spine_set_logical_compaction(s: *mut Spine, frontier: u64) -> i32;
    pub fn mzgpu_spine_set_physical_compaction(s: *mut Spine, frontier: u64) -> i32;
    pub fn mzgpu_spine_get_logical_compaction(s: *const Spine) -> u64;
    pub fn mzgpu_spine_get_physical_compaction(s: *const Spine) -> u64;
    pub fn mzgpu_spine_read_upper(s: *const Spine) -> u64;
    pub fn mzgpu_spine_batches_through(s: *mut Spine, upper: u64, batches: *mut *mut Batch, cap: u32, n_out: *mut u32) -> i32;
    pub fn mzgpu_spine_size(s: *const Spine, out: *mut ArrangementSize) -> i32;
    // a9, a10: joins
    pub fn mzgpu_join_new(ctx: *mut Ctx, t1: *mut Spine, t2: *mut Spine, c: *const Closure, out: *mut *mut Join) -> i32;
    pub fn mzgpu_join_free(j: *mut Join);
    pub fn mzgpu_join_core_push(j: *mut Join, side: i32, batch: *mut Batch, cap: u64) -> i32;
    pub fn mzgpu_join_core_work_until(j: *mut Join, fuel_rows: u64, deadline_ns: u64, out: *mut Buf, done: *mut i32) -> i32;
    pub fn mzgpu_half_join(ctx: *mut Ctx, stream: *const R32, n: u64, mem: i32, trace: *mut Spine, cmp_mode: i32,
                           closure: *const Closure, consolidate: i32, out: *mut Buf) -> i32;
    // a11, a12: reduce
    pub fn mzgpu_reduce_new(ctx: *mut Ctx, agg_kind: i32, out: *mut *mut Reduce) -> i32;
    pub fn mzgpu_reduce_free(r: *mut Reduce);
    pub fn mzgpu_reduce_accumulable(r: *mut Reduce, rows: *const R32, n: u64, mem: i32, upper: u64, out: *mut Buf) -> i32;
    // buffers
    pub fn mzgpu_buf_new(ctx: *mut Ctx, row_bytes: u32, out: *mut *mut Buf) -> i32;
    pub fn mzgpu_buf_free(b: *mut Buf);
    pub fn mzgpu_buf_len(b: *mut Buf) -> u64;
    pub fn mzgpu_buf_download(b: *mut Buf, rows: *mut c_void, cap: u64, mem: i32, n_out: *mut u64) -> i32;
    pub fn mzgpu_buf_clear(b: *mut Buf) -> i32;
    // f4: the columnar wire format (Column<C>)
    pub fn mzgpu_column_length_in_words(layout: i32, rows: u64, key_bytes: u64, val_bytes: u64) -> u64;
    pub fn mzgpu_column_at_capacity(words: u64) -> i32;
    pub fn mzgpu_column_ship_rows(layout: i32) -> u64;
    pub fn mzgpu_column_decode(ctx: *mut Ctx, layout: i32, words: *const u64, n_words: u64, mem: i32, out: *mut Buf) -> i32;
    pub fn mzgpu_column_encode(rows: *mut Buf, layout: i32, first: u64, n: u64, words: *mut u64, cap_words: u64, mem: i32,
                               n_words: *mut u64) -> i32;
    pub fn mzgpu_column_build(rows: *mut Buf, layout: i32, words: *mut u64, cap_words: u64, mem: i32, n_words: *mut u64,
                              chunk_words: *mut u64, cap_chunks: u32, n_chunks: *mut u32) -> i32;
    pub fn mzgpu_batch_walk_column(batch: *mut Batch, key: *const u64, first: u64, fuel: u64, layout: i32, words: *mut u64,
                                   cap_words: u64, mem: i32, n_words: *mut u64, n_rows: *mut u64) -> i32;
    pub fn mzgpu_batcher_push_buf(b: *mut Batcher, rows: *mut Buf) -> i32;
    pub fn mzgpu_buf_upload(b: *mut Buf, rows: *const c_void, n: u64, mem: i32) -> i32;
    // row L: linear join plans
    pub fn mzgpu_linear_join_new(ctx: *mut Ctx, plan: *const LinearJoinPlan, lookup_traces: *const *mut Spine,
                                 out: *mut *mut LinearJoin) -> i32;
    pub fn mzgpu_linear_join_free(lj: *mut LinearJoin);
    pub fn mzgpu_linear_join_step(lj: *mut LinearJoin, source: *mut Buf, lookup_batches: *const *mut Batch, upper: u64,
                                  out: *mut Buf) -> i32;
    pub fn mzgpu_linear_join_stage_trace(lj: *mut LinearJoin, stage: u32) -> *mut Spine;
    // ---- the rest of include/mzgpu.h, one to one (tests/test_abi.py::test_rust_shim_declares_every_entry_point)
    pub fn mzgpu_ctx_stats(ctx: *mut Ctx, out: *mut Stats) -> i32;
    pub fn mzgpu_ctx_host_times(ctx: *mut Ctx, out: *mut u64) -> i32;
    pub fn mzgpu_profile_enable(ctx: *mut Ctx, on: i32) -> i32;
    pub fn mzgpu_profile_report(ctx: *mut Ctx, buf: *mut c_char, cap: u64) -> i32;
    pub fn mzgpu_profile_fused_phases(ctx: *mut Ctx, out: *mut u64, cap_records: u32, n: *mut u32) -> i32;
    pub fn mzgpu_ctx_stream(ctx: *mut Ctx) -> *mut c_void;
    pub fn mzgpu_buf_row_bytes(buf: *const Buf) -> u32;
    pub fn mzgpu_buf_device_ptr(buf: *mut Buf) -> *mut c_void;
    pub fn mzgpu_buf_append(buf: *mut Buf, rows: *const c_void, n: u64, mem: i32) -> i32;
    pub fn mzgpu_buf_append_buf(dst: *mut Buf, src: *mut Buf) -> i32;
    pub fn mzgpu_buf_append_buf_at_most(dst: *mut Buf, src: *mut Buf, max_rows: u64) -> i32;
    pub fn mzgpu_consolidate_r16(ctx: *mut Ctx, rows: *mut R16, n: u64, mem: i32, n_out: *mut u64) -> i32;
    pub fn mzgpu_consolidate_r32(ctx: *mut Ctx, rows: *mut R32, n: u64, mem: i32, n_out: *mut u64) -> i32;
    pub fn mzgpu_buf_consolidate(buf: *mut Buf) -> i32;
    pub fn mzgpu_batcher_seal_many(k: u32, batchers: *const *mut Batcher, upper: u64, batches_out: *mut *mut Batch) -> i32;
    pub fn mzgpu_batcher_len(b: *const Batcher) -> u64;
    pub fn mzgpu_batch_build(ctx: *mut Ctx, row_bytes: u32, rows: *const c_void, n: u64, mem: i32, desc: Desc, out: *mut *mut Batch) -> i32;
    pub fn mzgpu_batch_export(b: *mut Batch, rows: *mut c_void, cap: u64, mem: i32, n_out: *mut u64) -> i32;
    pub fn mzgpu_builder_push_buf(b: *mut Builder, rows: *mut Buf) -> i32;
    pub fn mzgpu_spine_layers(s: *const Spine, out4: *mut u64, cap_layers: u32, n_layers: *mut u32) -> i32;
    pub fn mzgpu_spine_export(s: *mut Spine, out: *mut Buf) -> i32;
    pub fn mzgpu_join_core_work(j: *mut Join, fuel_rows: u64, out: *mut Buf, done: *mut i32) -> i32;
    pub fn mzgpu_half_join_buf(ctx: *mut Ctx, stream: *mut Buf, trace: *mut Spine, cmp_mode: i32, closure: *const Closure, consolidate_output: i32, out: *mut Buf) -> i32;
    pub fn mzgpu_half_join_many(ctx: *mut Ctx, k: u32, streams: *const *mut Buf, traces: *const *mut Spine, cmp_modes: *const i32, closures: *const *const Closure, outs: *const *mut Buf) -> i32;
    pub fn mzgpu_delta_first_stage_many(ctx: *mut Ctx, k: u32, batches: *const *mut Batch, initial_closures: *const *const Closure, skip_times: *const u64, traces: *const *mut Spine, cmp_modes: *const i32, closures: *const *const Closure, outs: *const *mut Buf) -> i32;
    pub fn mzgpu_update_stream(ctx: *mut Ctx, batch: *mut Batch, initial_closure: *const Closure, skip_time: u64, out: *mut Buf) -> i32;
    pub fn mzgpu_map_rows(ctx: *mut Ctx, rows: *const R32, n: u64, mem: i32, closure: *const Closure, out: *mut Buf) -> i32;
    pub fn mzgpu_topk_new(ctx: *mut Ctx, limit: i64, offset: u64, descending: i32, out: *mut *mut Reduce) -> i32;
    pub fn mzgpu_reduce_accumulable_buf(r: *mut Reduce, rows: *mut Buf, upper: u64, out: *mut Buf) -> i32;
    pub fn mzgpu_reduce_input_trace(r: *mut Reduce) -> *mut Spine;
    pub fn mzgpu_reduce_lanes_row_bytes(n_lanes: u32, arr_row_bytes: *mut u32, out_row_bytes: *mut u32) -> i32;
    pub fn mzgpu_reduce_lanes_new(ctx: *mut Ctx, in_row_bytes: u32, lanes: *const AccumLane, n_lanes: u32, out: *mut *mut Reduce) -> i32;
    pub fn mzgpu_reduce_lanes(r: *mut Reduce, rows: *const c_void, n: u64, mem: i32, upper: u64, out: *mut Buf) -> i32;
    pub fn mzgpu_reduce_lanes_buf(r: *mut Reduce, rows: *mut Buf, upper: u64, out: *mut Buf) -> i32;
    pub fn mzgpu_reduce_lanes_distinct_trace(r: *mut Reduce, lane: u32) -> *mut Spine;
    pub fn mzgpu_rowkey_pack(row_bytes: *const u8, len: u64, key_out: *mut u64) -> i32;
    pub fn mzgpu_rowkeys_pack(data: *const u8, offsets: *const u64, n: u64, keys_out: *mut u64, n_done: *mut u64) -> i32;
    pub fn mzgpu_rowkey_unpack(key: u64, row_bytes_out: *mut u8, len_out: *mut u64) -> i32;
    pub fn mzgpu_correction_new(ctx: *mut Ctx, out: *mut *mut Correction) -> i32;
    pub fn mzgpu_correction_free(c: *mut Correction);
    pub fn mzgpu_correction_insert(c: *mut Correction, rows: *const R32, n: u64, mem: i32, negate: i32) -> i32;
    pub fn mzgpu_correction_insert_buf(c: *mut Correction, rows: *mut Buf, negate: i32) -> i32;
    pub fn mzgpu_correction_updates_before(c: *mut Correction, upper: u64, out: *mut Buf) -> i32;
    pub fn mzgpu_correction_advance_since(c: *mut Correction, since: u64) -> i32;
    pub fn mzgpu_correction_consolidate_at_since(c: *mut Correction) -> i32;
    pub fn mzgpu_correction_len(c: *mut Correction) -> u64;
    pub fn mzgpu_comm_unique_id(id: *mut u8) -> i32;
    pub fn mzgpu_comm_init(ctx: *mut Ctx, id: *const u8) -> i32;
    pub fn mzgpu_exchange(ctx: *mut Ctx, input: *mut Buf, out: *mut Buf) -> i32;
    pub fn mzgpu_exchange_many(ctx: *mut Ctx, k: u32, ins: *mut *mut Buf, outs: *mut *mut Buf) -> i32;
    pub fn mzgpu_comm_p2p_export(ctx: *mut Ctx, landing_rows: u64, region_row_bytes: u32, handle: *mut u8) -> i32;
    pub fn mzgpu_comm_p2p_import(ctx: *mut Ctx, handles: *const u8) -> i32;
    pub fn mzgpu_comm_p2p_zone(ctx: *mut Ctx) -> *mut c_void;
    pub fn mzgpu_comm_p2p_import_local(ctx: *mut Ctx, zones: *const *mut c_void) -> i32;
    pub fn mzgpu_exchange_p2p(ctx: *mut Ctx, k: u32, ins: *mut *mut Buf, outs: *mut *mut Buf, recv_ub: *const u64) -> i32;
    pub fn mzgpu_exchange_p2p_send(ctx: *mut Ctx, k: u32, ins: *mut *mut Buf) -> i32;
    pub fn mzgpu_exchange_p2p_recv(ctx: *mut Ctx, k: u32, outs: *mut *mut Buf, recv_ub: *const u64) -> i32;
    pub fn mzgpu_route(key: u64, peers: u32) -> u32;
    pub fn mzgpu_partition_many(ctx: *mut Ctx, k: u32, ins: *mut *mut Buf, peers: u32, outs: *mut *mut Buf, counts: *mut u64) -> i32;
}
pub enum LinearJoin {}
pub const LINEAR_MAX_STAGES: usize = 6;
#[repr(C)] pub struct LinearStagePlan { pub stream_key: Closure, pub closure: Closure }
#[repr(C)] pub struct LinearJoinPlan {
    pub has_initial_closure: i32, pub has_final_closure: i32, pub n_stages: u32, pub _pad: u32,
    pub initial_closure: Closure, pub final_closure: Closure, pub stages: [LinearStagePlan; LINEAR_MAX_STAGES],
}
pub const COLUMN_U64X4: i32 = 0;
pub const COLUMN_U64X2: i32 = 1;
pub const COLUMN_ROWROW: i32 = 2;

/// Status -> Result; CUDA / NCCL failures are sticky: the caller panics the worker (compute state
/// is soft, the replica rehydrates: src/cluster/src/communication.rs:18-27).
pub unsafe fn check(ctx: *mut Ctx, st: i32) -> Result<(), (i32, String)> {
    if st == OK { return Ok(()); }
    let msg = std::ffi::CStr::from_ptr(mzgpu_last_error(ctx)).to_string_lossy().into_owned();
    if st == E_CUDA || st == E_NCCL { panic!("mzgpu: sticky device failure {st}: {msg}"); }
    Err((st, msg))
}
