//! Temporal filters: `Plan::Mfp` / `GetPlan::*(mfp)` with `mz_now()` bounds (MfpPlan, src/expr/src/linear.rs),
//! rendered by `as_collection_core` (src/compute/src/render/context.rs:895-975), with the future updates held
//! on the device until the frontier reaches them (the temporal delay operator's bucket chain).
use crate::sys;
use crate::worker_ctx;

pub struct GpuMfp { h: *mut sys::MfpOp }

impl GpuMfp {
    /// MZGPU_E_UNSUPPORTED: keep the Rust operator for this plan.
    pub fn new(plan: &sys::Mfp, until: u64) -> Result<Self, (i32, String)> {
        let mut h = std::ptr::null_mut();
        unsafe { sys::check(worker_ctx(), sys::mzgpu_mfp_new(worker_ctx(), plan, until, &mut h))?; }
        Ok(GpuMfp { h })
    }
    /// The plan with map expressions (`MapFilterProject::expressions`, or a `KeyValPlan`'s key and value
    /// expressions): predicates, temporal programs and output fields read them.  MZGPU_E_UNSUPPORTED: keep the
    /// Rust operator for this plan.
    pub fn new_map(plan: &sys::Mfp, map: &sys::MfpMap, until: u64) -> Result<Self, (i32, String)> {
        let mut h = std::ptr::null_mut();
        unsafe { sys::check(worker_ctx(), sys::mzgpu_mfp_new_map(worker_ctx(), plan, map, until, &mut h))?; }
        Ok(GpuMfp { h })
    }
    /// One activation: updates due before `upper` (new and held) are appended to `out`, consolidated; errors
    /// (R32: code, payload, time, diff) to `errs`.
    pub fn step(&mut self, rows: *mut sys::Buf, upper: u64, out: *mut sys::Buf, errs: *mut sys::Buf) -> Result<(), (i32, String)> {
        unsafe { sys::check(worker_ctx(), sys::mzgpu_mfp_step_buf(self.h, rows, upper, out, errs)) }
    }
    /// The least held time (u64::MAX: nothing held): the operator's capability is held there.  An error
    /// leaves the capability where it was.
    pub fn frontier(&self) -> Result<u64, (i32, String)> {
        let mut t = 0u64;
        unsafe { sys::check(worker_ctx(), sys::mzgpu_mfp_frontier(self.h, &mut t))?; }
        Ok(t)
    }
    /// (held rows, buckets, rows the store touched in the last step).
    pub fn stats(&self) -> Result<[u64; 3], (i32, String)> {
        let mut a = [0u64; 3];
        unsafe { sys::check(worker_ctx(), sys::mzgpu_mfp_stats(self.h, a.as_mut_ptr()))?; }
        Ok(a)
    }
}

impl Drop for GpuMfp {
    fn drop(&mut self) { unsafe { sys::mzgpu_mfp_free(self.h) } }
}
