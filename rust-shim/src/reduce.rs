//! `mz_reduce_abelian` instances over a device arrangement.  UNCOMPILED: see ../README.md.
//!
//! One handle covers the plans of src/compute/src/render/reduce.rs that are reductions of an
//! arrangement with an abelian diff: accumulable COUNT/SUM (`build_accumulable`, :1261-1471: explode
//! into the `Accum` semigroup, arrange, `reduce_abelian`, `finalize_accum` :1575-1584,1671-1700),
//! DISTINCT (`build_distinct`, :264-334), threshold (src/compute/src/render/threshold.rs:33-77),
//! MIN / MAX (`build_bucketed_negated_output`, :1050-1135) and TopK (`BasicTopKPlan`,
//! src/compute/src/render/top_k.rs:215-248).  An activation takes the input updates that arrived
//! (device buffer or host slice), seals the operator's own input arrangement at `upper` and appends
//! the output corrections (`sys::Rout`) — the `(key, aggregates) +-1` rows `reduce_abelian` emits.
use super::sys::{self, R32};
use super::worker_ctx;

pub enum ReduceKind {
    CountSumI64, CountSumF64, Distinct, Threshold, Min, Max,
    /// `limit < 0`: LIMIT NULL
    TopK { limit: i64, offset: u64, descending: bool },
}

pub struct GpuReduce { h: *mut sys::Reduce }

impl GpuReduce {
    pub fn new(kind: ReduceKind) -> Result<Self, (i32, String)> {
        let mut h = std::ptr::null_mut();
        let st = unsafe {
            match kind {
                ReduceKind::TopK { limit, offset, descending } =>
                    sys::mzgpu_topk_new(worker_ctx(), limit, offset, descending as i32, &mut h),
                k => sys::mzgpu_reduce_new(worker_ctx(), match k {
                    ReduceKind::CountSumI64 => sys::AGG_COUNT_SUM_I64,
                    ReduceKind::CountSumF64 => sys::AGG_COUNT_SUM_F64,
                    ReduceKind::Distinct => sys::AGG_DISTINCT,
                    ReduceKind::Threshold => sys::AGG_THRESHOLD,
                    ReduceKind::Min => sys::AGG_MIN,
                    _ => sys::AGG_MAX,
                }, &mut h),
            }
        };
        // plans the device subset cannot hold (a TopK window wider than 32 on a wide group, ...)
        // come back as E_UNSUPPORTED: the caller renders the Rust operator instead
        unsafe { sys::check(worker_ctx(), st)?; }
        Ok(GpuReduce { h })
    }
    /// One activation over host updates `((key, val), time, diff)`.
    pub fn step_host(&mut self, updates: &[((u64, u64), u64, i64)], upper: u64, out: *mut sys::Buf) -> Result<(), (i32, String)> {
        let st = unsafe {
            sys::mzgpu_reduce_accumulable(self.h, updates.as_ptr() as *const R32, updates.len() as u64, sys::MEM_HOST, upper, out)
        };
        unsafe { sys::check(worker_ctx(), st) }
    }
    /// One activation over a device buffer (the result collection of a delta / linear join): the
    /// row count stays on the device, nothing is read back.
    pub fn step(&mut self, rows: *mut sys::Buf, upper: u64, out: *mut sys::Buf) -> Result<(), (i32, String)> {
        unsafe { sys::check(worker_ctx(), sys::mzgpu_reduce_accumulable_buf(self.h, rows, upper, out)) }
    }
    /// The operator's input arrangement (for compaction: `TraceManager::maintenance`,
    /// src/compute/src/arrangement/manager.rs:55-73).
    pub fn input_trace(&self) -> *mut sys::Spine { unsafe { sys::mzgpu_reduce_input_trace(self.h) } }
}
/// `build_accumulable` over several aggregates (`AccumulablePlan::simple_aggrs`, reduce.rs:146-158 of
/// src/compute-types/src/plan): one arrangement of `(Vec<Accum>, Diff)`, one output row per key with
/// every lane's COUNT and SUM (`sys::mzgpu_reduce_lanes_new` documents the row layouts).  The input is
/// R32 (`in_row_bytes` 32) or a join's R40 result (40).  An int64 lane whose kind carries
/// `sys::ACCUM_DISTINCT` is one of the plan's `distinct_aggrs`; a float64 distinct lane comes back as
/// `MZGPU_E_UNSUPPORTED`, so the caller keeps the Rust operator for such plans.
pub struct GpuReduceLanes { h: *mut sys::Reduce, pub arr_row_bytes: u32, pub out_row_bytes: u32 }

impl GpuReduceLanes {
    pub fn new(in_row_bytes: u32, lanes: &[sys::AccumLane]) -> Result<Self, (i32, String)> {
        let (mut arr, mut out) = (0u32, 0u32);
        let mut h = std::ptr::null_mut();
        unsafe {
            sys::check(worker_ctx(), sys::mzgpu_reduce_lanes_row_bytes(lanes.len() as u32, &mut arr, &mut out))?;
            sys::check(worker_ctx(), sys::mzgpu_reduce_lanes_new(worker_ctx(), in_row_bytes, lanes.as_ptr(), lanes.len() as u32, &mut h))?;
        }
        Ok(GpuReduceLanes { h, arr_row_bytes: arr, out_row_bytes: out })
    }
    /// The same with the filter half of the reduce's `mfp_after` (`sys::Having`, INTEGRATION.md maps a
    /// `SafeMfpPlan`'s predicates to it).  A program outside the device subset comes back as
    /// `MZGPU_E_UNSUPPORTED`: the caller keeps the Rust operator for that plan.
    pub fn new_having(in_row_bytes: u32, lanes: &[sys::AccumLane], having: &sys::Having) -> Result<Self, (i32, String)> {
        let (mut arr, mut out) = (0u32, 0u32);
        let mut h = std::ptr::null_mut();
        unsafe {
            sys::check(worker_ctx(), sys::mzgpu_reduce_lanes_row_bytes(lanes.len() as u32, &mut arr, &mut out))?;
            sys::check(worker_ctx(), sys::mzgpu_reduce_lanes_new_having(worker_ctx(), in_row_bytes, lanes.as_ptr(),
                                                                       lanes.len() as u32, having, &mut h))?;
        }
        Ok(GpuReduceLanes { h, arr_row_bytes: arr, out_row_bytes: out })
    }
    /// One activation over a device buffer of input rows; output rows (`out_row_bytes` wide) are appended to `out`.
    pub fn step(&mut self, rows: *mut sys::Buf, upper: u64, out: *mut sys::Buf) -> Result<(), (i32, String)> {
        unsafe { sys::check(worker_ctx(), sys::mzgpu_reduce_lanes_buf(self.h, rows, upper, out)) }
    }
    pub fn input_trace(&self) -> *mut sys::Spine { unsafe { sys::mzgpu_reduce_input_trace(self.h) } }
    /// The (key, value) pair arrangement of distinct lane `lane` ("Arranged Accumulable Distinct"); null
    /// for any other lane.
    pub fn distinct_trace(&self, lane: u32) -> *mut sys::Spine {
        unsafe { sys::mzgpu_reduce_lanes_distinct_trace(self.h, lane) }
    }
}
impl Drop for GpuReduceLanes {
    fn drop(&mut self) { unsafe { sys::mzgpu_reduce_free(self.h) } }
}

/// `build_monotonic` (`HierarchicalPlan::Monotonic`, reduce.rs:160-250 of src/compute-types/src/plan; the
/// planner's choice for append-only inputs): several MIN / MAX aggregates per key, the best value of each
/// kept in the arrangement's diff (`sys::mzgpu_reduce_monotonic_new` documents the row layouts and the lane
/// encoding).  Lanes are `sys::AccumLane`s of kind `AGG_MIN` / `AGG_MAX`; `sign_extend != 0` is signed
/// order.  `must_consolidate` is the plan's flag.  A float64 lane (`sys::MONO_F64`) comes back as
/// `MZGPU_E_UNSUPPORTED`, and so does nothing else: the caller keeps the Rust operator for such plans and
/// for an `mfp_after` with a filter.
pub struct GpuReduceMonotonic { h: *mut sys::Reduce, pub arr_row_bytes: u32, pub out_row_bytes: u32 }

impl GpuReduceMonotonic {
    pub fn new(in_row_bytes: u32, lanes: &[sys::AccumLane], must_consolidate: bool) -> Result<Self, (i32, String)> {
        let (mut arr, mut out) = (0u32, 0u32);
        let mut h = std::ptr::null_mut();
        unsafe {
            sys::check(worker_ctx(), sys::mzgpu_reduce_monotonic_row_bytes(lanes.len() as u32, &mut arr, &mut out))?;
            sys::check(worker_ctx(), sys::mzgpu_reduce_monotonic_new(worker_ctx(), in_row_bytes, lanes.as_ptr(),
                                                                    lanes.len() as u32, must_consolidate as i32, &mut h))?;
        }
        Ok(GpuReduceMonotonic { h, arr_row_bytes: arr, out_row_bytes: out })
    }
    /// One activation over a device buffer of input rows: corrections (`out_row_bytes` wide) are appended to
    /// `out`, the `ensure_monotonic` errors (R16: time, count) to `errs`.
    pub fn step(&mut self, rows: *mut sys::Buf, upper: u64, out: *mut sys::Buf, errs: *mut sys::Buf) -> Result<(), (i32, String)> {
        unsafe { sys::check(worker_ctx(), sys::mzgpu_reduce_monotonic_buf(self.h, rows, upper, out, errs)) }
    }
    pub fn input_trace(&self) -> *mut sys::Spine { unsafe { sys::mzgpu_reduce_input_trace(self.h) } }
}
impl Drop for GpuReduceMonotonic {
    fn drop(&mut self) { unsafe { sys::mzgpu_reduce_free(self.h) } }
}

/// `build_bucketed` (`HierarchicalPlan::Bucketed`, reduce.rs:232-250 of src/compute-types/src/plan; the
/// planner's choice for MIN / MAX over a collection that can retract): several MIN / MAX aggregates per key,
/// one output row per key (`sys::mzgpu_reduce_hierarchical_new` documents the semantics and the rows).  Lanes
/// are `sys::AccumLane`s of kind `AGG_MIN` / `AGG_MAX`; `sign_extend != 0` is signed order.  A float64 lane
/// (`sys::MONO_F64`) comes back as `MZGPU_E_UNSUPPORTED`: the caller keeps the Rust operator for such plans.
pub struct GpuReduceHierarchical { h: *mut sys::Reduce, pub out_row_bytes: u32 }

impl GpuReduceHierarchical {
    pub fn new(in_row_bytes: u32, lanes: &[sys::AccumLane]) -> Result<Self, (i32, String)> {
        let mut out = 0u32;
        let mut h = std::ptr::null_mut();
        unsafe {
            sys::check(worker_ctx(), sys::mzgpu_reduce_monotonic_row_bytes(lanes.len() as u32, std::ptr::null_mut(), &mut out))?;
            sys::check(worker_ctx(), sys::mzgpu_reduce_hierarchical_new(worker_ctx(), in_row_bytes, lanes.as_ptr(),
                                                                       lanes.len() as u32, &mut h))?;
        }
        Ok(GpuReduceHierarchical { h, out_row_bytes: out })
    }
    /// One activation over a device buffer of input rows: corrections (`out_row_bytes` wide) are appended to
    /// `out`, the non-positive-accumulation errors (R32: key, 0, time, +1 / -1) to `errs`.
    pub fn step(&mut self, rows: *mut sys::Buf, upper: u64, out: *mut sys::Buf, errs: *mut sys::Buf) -> Result<(), (i32, String)> {
        unsafe { sys::check(worker_ctx(), sys::mzgpu_reduce_hierarchical_buf(self.h, rows, upper, out, errs)) }
    }
    /// The arrangement of the masked input rows (R32 / R40, the input width).
    pub fn input_trace(&self) -> *mut sys::Spine { unsafe { sys::mzgpu_reduce_input_trace(self.h) } }
}
impl Drop for GpuReduceHierarchical {
    fn drop(&mut self) { unsafe { sys::mzgpu_reduce_free(self.h) } }
}

/// `TopKPlan::MonotonicTop1` / `MonotonicTopK` (top_k.rs:102-214 of src/compute/src/render): the first
/// `limit` rows per key of an append-only input, with only that window arranged
/// (`sys::mzgpu_topk_monotonic_new` documents the order and the window rows).  Top1 is `limit = 1`;
/// `LIMIT NULL` is `sys::TOPK_NO_LIMIT`.  A negative literal limit or a float64 order column
/// (`sys::ORDER_F64`) comes back as `MZGPU_E_UNSUPPORTED`: the caller keeps the Rust operator for those,
/// and for a limit given as an expression.
pub struct GpuTopKMonotonic { h: *mut sys::Reduce }

impl GpuTopKMonotonic {
    pub fn new(in_row_bytes: u32, order: &[sys::OrderLane], limit: i64, must_consolidate: bool) -> Result<Self, (i32, String)> {
        let mut h = std::ptr::null_mut();
        unsafe {
            sys::check(worker_ctx(), sys::mzgpu_topk_monotonic_new(worker_ctx(), in_row_bytes, order.as_ptr(),
                                                                  order.len() as u32, limit, must_consolidate as i32, &mut h))?;
        }
        Ok(GpuTopKMonotonic { h })
    }
    /// One activation over a device buffer of input rows: the window changes (input-width rows) are appended
    /// to `out`, the `ensure_monotonic` errors (R16: time, count) to `errs`.
    pub fn step(&mut self, rows: *mut sys::Buf, upper: u64, out: *mut sys::Buf, errs: *mut sys::Buf) -> Result<(), (i32, String)> {
        unsafe { sys::check(worker_ctx(), sys::mzgpu_topk_monotonic_buf(self.h, rows, upper, out, errs)) }
    }
    /// The window arrangement (72-byte rows), compacted by the caller like any other trace.
    pub fn window_trace(&self) -> *mut sys::Spine { unsafe { sys::mzgpu_reduce_input_trace(self.h) } }
}
impl Drop for GpuTopKMonotonic {
    fn drop(&mut self) { unsafe { sys::mzgpu_reduce_free(self.h) } }
}

/// `BasicTopKPlan` (`build_topk` / `build_topk_negated_stage`): whole rows over input that retracts, with an
/// OFFSET (`sys::mzgpu_topk_basic_new` documents the order, the window and the error rows).  Each `ColumnOrder`
/// is one order lane; `LIMIT NULL` is `sys::TOPK_NO_LIMIT`.  A negative literal limit, a float64 order column,
/// or `offset + limit` past `i64::MAX` comes back as `MZGPU_E_UNSUPPORTED`: the caller keeps the Rust operator
/// for those, and for a limit given as an expression.
pub struct GpuTopKBasic { h: *mut sys::Reduce }

impl GpuTopKBasic {
    pub fn new(in_row_bytes: u32, order: &[sys::OrderLane], limit: i64, offset: u64) -> Result<Self, (i32, String)> {
        let mut h = std::ptr::null_mut();
        unsafe {
            sys::check(worker_ctx(), sys::mzgpu_topk_basic_new(worker_ctx(), in_row_bytes, order.as_ptr(),
                                                              order.len() as u32, limit, offset, &mut h))?;
        }
        Ok(GpuTopKBasic { h })
    }
    /// One activation over a device buffer of input rows: the window changes (input-width rows) are appended
    /// to `out`, the error-state changes (R32: key, 0, time, +1 / -1) to `errs`, the error collection.
    pub fn step(&mut self, rows: *mut sys::Buf, upper: u64, out: *mut sys::Buf, errs: *mut sys::Buf) -> Result<(), (i32, String)> {
        unsafe { sys::check(worker_ctx(), sys::mzgpu_topk_basic_buf(self.h, rows, upper, out, errs)) }
    }
    /// The input arrangement (72-byte rows), compacted by the caller like any other trace.
    pub fn input_trace(&self) -> *mut sys::Spine { unsafe { sys::mzgpu_reduce_input_trace(self.h) } }
    /// The negatives arrangement (R32), compacted by the operator itself; for inspection and size logging.
    pub fn negatives_trace(&self) -> *mut sys::Spine { unsafe { sys::mzgpu_topk_basic_negatives_trace(self.h) } }
}

impl Drop for GpuTopKBasic {
    fn drop(&mut self) { unsafe { sys::mzgpu_reduce_free(self.h) } }
}

impl Drop for GpuReduce {
    fn drop(&mut self) { unsafe { sys::mzgpu_reduce_free(self.h) } }
}
