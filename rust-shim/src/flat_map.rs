//! FlatMap: `Plan::FlatMap` (src/compute/src/render.rs:1240-1249), rendered by `render_flat_map`
//! (src/compute/src/render/flat_map.rs:29-200) for generate_series, repeat_row and the subquery size guard: the
//! table function's rows are expanded on the device in pages of `fuel` function rows and run through the MfpPlan,
//! whose future updates are held on the device as `GpuMfp` holds them.
use crate::sys;
use crate::worker_ctx;

pub struct GpuFlatMap { h: *mut sys::FlatMapOp }

impl GpuFlatMap {
    /// MZGPU_E_UNSUPPORTED: keep the Rust operator for this table function or plan.
    pub fn new(func: &sys::TableFunc, plan: &sys::Mfp, map: Option<&sys::MfpMap>, until: u64) -> Result<Self, (i32, String)> {
        let mut h = std::ptr::null_mut();
        let map = map.map_or(std::ptr::null(), |m| m as *const sys::MfpMap);
        unsafe { sys::check(worker_ctx(), sys::mzgpu_flat_map_new(worker_ctx(), func, plan, map, until, &mut h))?; }
        Ok(GpuFlatMap { h })
    }
    /// One activation of the `FlatMapStage` operator: the input container's rows, expanded `fuel` function rows at a
    /// time (COMPUTE_FLAT_MAP_FUEL) until done.  Each page appends its due updates to `out` and its errors to
    /// `errs`, consolidated; between pages the caller may yield and re-activate itself, as the reference does
    /// between containers.
    pub fn activate(&mut self, rows: *mut sys::Buf, upper: u64, fuel: u64, out: *mut sys::Buf, errs: *mut sys::Buf,
                    mut yield_now: impl FnMut() -> bool) -> Result<bool, (i32, String)> {
        let mut done = 0i32;
        unsafe { sys::check(worker_ctx(), sys::mzgpu_flat_map_step_buf(self.h, rows, upper, fuel, out, errs, &mut done))?; }
        while done == 0 {
            if yield_now() {
                return Ok(false);
            }
            unsafe { sys::check(worker_ctx(), sys::mzgpu_flat_map_work(self.h, fuel, out, errs, &mut done))?; }
        }
        Ok(true)
    }
    /// Continue an activation that `activate` left unfinished (`Ok(false)`): true once it is done.
    pub fn work(&mut self, fuel: u64, out: *mut sys::Buf, errs: *mut sys::Buf) -> Result<bool, (i32, String)> {
        let mut done = 0i32;
        unsafe { sys::check(worker_ctx(), sys::mzgpu_flat_map_work(self.h, fuel, out, errs, &mut done))?; }
        Ok(done != 0)
    }
    /// Where the operator holds its capability: the least held time, or during an activation the least time of
    /// the rows not yet expanded if lower (u64::MAX: nothing).
    pub fn frontier(&self) -> Result<u64, (i32, String)> {
        let mut t = 0u64;
        unsafe { sys::check(worker_ctx(), sys::mzgpu_flat_map_frontier(self.h, &mut t))?; }
        Ok(t)
    }
    /// (held rows, buckets, rows the store touched in the last page, function rows still to expand).
    pub fn stats(&self) -> Result<[u64; 4], (i32, String)> {
        let mut a = [0u64; 4];
        unsafe { sys::check(worker_ctx(), sys::mzgpu_flat_map_stats(self.h, a.as_mut_ptr()))?; }
        Ok(a)
    }
}

impl Drop for GpuFlatMap {
    fn drop(&mut self) { unsafe { sys::mzgpu_flat_map_free(self.h) } }
}
