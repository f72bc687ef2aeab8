//! `LinearJoinImpl::Gpu` — a rendered `LinearJoinPlan` on the device.  UNCOMPILED: see ../README.md.
//!
//! `LinearJoinSpec::render` (src/compute/src/render/join/linear_join.rs:109-132) dispatches on
//! `LinearJoinImpl`; a third variant lowers the plan (src/compute-types/src/plan/join/linear_join.rs:26-62)
//! to the POD descriptor of include/mzgpu.h when every key / thinning expression is a column pick on
//! fixed-width integer columns and every `JoinClosure` is projection + comparisons (plan lowering,
//! INTEGRATION.md §2 last row); anything else keeps the Materialize rendering (`MZGPU_E_UNSUPPORTED`
//! is a render-time answer, never a runtime fallback inside the operator).
use super::sys;
use super::worker_ctx;

pub struct GpuLinearJoin { h: *mut sys::LinearJoin, out: *mut sys::Buf, src: *mut sys::Buf }

impl GpuLinearJoin {
    /// `lookup_traces[s]` = the arrangement of stage s's lookup relation by its `lookup_key`
    /// (a `GpuSpine`'s handle): `inputs[stage_plan.lookup_relation].arrangement(&lookup_key)`,
    /// linear_join.rs:404-406.
    pub fn new(plan: &sys::LinearJoinPlan, lookup_traces: &[*mut sys::Spine]) -> Result<Self, (i32, String)> {
        let (mut h, mut out, mut src) = (std::ptr::null_mut(), std::ptr::null_mut(), std::ptr::null_mut());
        unsafe {
            sys::check(worker_ctx(), sys::mzgpu_linear_join_new(worker_ctx(), plan, lookup_traces.as_ptr(), &mut h))?;
            sys::check(worker_ctx(), sys::mzgpu_buf_new(worker_ctx(), sys::ROW_R32, &mut out))?;
            sys::check(worker_ctx(), sys::mzgpu_buf_new(worker_ctx(), sys::ROW_R32, &mut src))?;
        }
        Ok(GpuLinearJoin { h, out, src })
    }

    /// One operator activation: the source relation's new updates and, per stage, the batch that
    /// arrived on the lookup arrangement (null if none); returns the final collection's new updates.
    /// The operator closure built in `render` calls this when its input frontiers have advanced to
    /// `upper` and re-activates itself while a fuel-limited variant reports work left.
    pub fn step(&mut self, source: &[sys::R32], lookup_batches: &[*mut sys::Batch], upper: u64) -> Vec<sys::R32> {
        unsafe {
            sys::check(worker_ctx(), sys::mzgpu_buf_upload(self.src, source.as_ptr() as *const _, source.len() as u64, sys::MEM_HOST)).expect("upload");
            sys::check(worker_ctx(), sys::mzgpu_buf_clear(self.out)).expect("clear");
            sys::check(worker_ctx(), sys::mzgpu_linear_join_step(self.h, self.src, lookup_batches.as_ptr(), upper, self.out)).expect("linear_join_step");
            let n = sys::mzgpu_buf_len(self.out);
            let mut rows = vec![sys::R32::default(); n as usize];
            let mut got = 0u64;
            sys::check(worker_ctx(), sys::mzgpu_buf_download(self.out, rows.as_mut_ptr() as *mut _, n, sys::MEM_HOST, &mut got)).expect("download");
            rows
        }
    }
}

impl Drop for GpuLinearJoin {
    fn drop(&mut self) {
        unsafe { sys::mzgpu_linear_join_free(self.h); sys::mzgpu_buf_free(self.out); sys::mzgpu_buf_free(self.src); }
    }
}

/// One join_core stage with a `JoinClosure` outside `mzgpu_closure`, composed by hand (the plan
/// descriptor takes bit-field closures only): `mzgpu_join_new_mfp` over the stream's and the lookup's
/// arrangements, then `work` per activation; error rows (R32) go to the error collection.
pub struct GpuJoinStageMfp { h: *mut sys::Join }

impl GpuJoinStageMfp {
    /// `jc` must outlive the stage.
    pub fn new(t1: *mut sys::Spine, t2: *mut sys::Spine, jc: *const sys::JoinClosure) -> Result<Self, (i32, String)> {
        let mut h = std::ptr::null_mut();
        unsafe { sys::check(worker_ctx(), sys::mzgpu_join_new_mfp(worker_ctx(), t1, t2, jc, &mut h))?; }
        Ok(GpuJoinStageMfp { h })
    }

    /// Work::process with the yield function: output and error rows count as fuel.  Returns done.
    pub fn work(&mut self, fuel: u64, deadline_ns: u64, out: *mut sys::Buf, errs: *mut sys::Buf) -> Result<bool, (i32, String)> {
        let mut done = 0i32;
        unsafe { sys::check(worker_ctx(), sys::mzgpu_join_core_work_mfp(self.h, fuel, deadline_ns, out, errs, &mut done))?; }
        Ok(done != 0)
    }
}

impl Drop for GpuJoinStageMfp {
    fn drop(&mut self) {
        unsafe { sys::mzgpu_join_free(self.h); }
    }
}
