//! Index peeks: `IndexPeek` (src/compute/src/compute_state.rs:1433-1673) answered on the device.  The worker lowers
//! `Peek { literal_constraints, map_filter_project, finishing, timestamp }` to a `PeekPlan` and a request
//! (INTEGRATION.md §2); a plan the lowering refuses (`MZGPU_E_UNSUPPORTED` / `_INVALID`) keeps the Rust peek.
use std::marker::PhantomData;

use crate::sys;
use crate::worker_ctx;

pub struct GpuPeek { h: *mut sys::PeekPlan }

impl GpuPeek {
    /// The `SafeMfpPlan` over the trace's (key, val) and the `RowSetFinishing`.  An error: keep the Rust peek.
    pub fn new(plan: &sys::Mfp, map: Option<&sys::MfpMap>, fin: &sys::Finishing) -> Result<Self, (i32, String)> {
        let mut h = std::ptr::null_mut();
        let map = map.map_or(std::ptr::null(), |m| m as *const _);
        unsafe { sys::check(worker_ctx(), sys::mzgpu_peek_plan_new(worker_ctx(), plan, map, fin, &mut h))?; }
        Ok(GpuPeek { h })
    }
    /// The request of this plan at `as_of`: `literals` None is a full scan; `max_rows` 0 is no limit.  The request
    /// borrows the plan and the literal keys for as long as it lives.
    pub fn request<'a>(&'a self, as_of: u64, literals: Option<&'a [u64]>, max_rows: u64) -> PeekRequest<'a> {
        let (p, n) = literals.map_or((std::ptr::null(), 0), |l| (l.as_ptr(), l.len() as u64));
        let req = sys::PeekReq { plan: self.h, as_of, literals: p, n_literals: n, literals_mem: sys::MEM_HOST, max_rows };
        PeekRequest { req, _borrows: PhantomData }
    }
}

/// An `mzgpu_peek_req` whose plan and literal keys outlive it (the same layout, so a slice of them is the C array).
#[repr(transparent)]
pub struct PeekRequest<'a> { req: sys::PeekReq, _borrows: PhantomData<(&'a GpuPeek, &'a [u64])> }

/// The pending peeks of one worker against one trace, answered in one call (at most `PEEK_MANY_MAX`): outs[i] gets
/// request i's rows when results[i].status is `PEEK_ROWS`; `PEEK_NOT_READY` stays pending, `PEEK_ERROR` becomes
/// `PeekResponse::Error`.
/// One output buffer per request: a length mismatch panics before the call.
pub fn peek_many(ok: *mut sys::Spine, errs: *mut sys::Spine, reqs: &[PeekRequest<'_>], outs: &[*mut sys::Buf])
                 -> Result<Vec<sys::PeekResult>, (i32, String)> {
    assert_eq!(reqs.len(), outs.len(), "peek_many: one output buffer per request");
    let mut res = vec![sys::PeekResult::default(); reqs.len()];
    unsafe {
        sys::check(worker_ctx(), sys::mzgpu_peek_many(worker_ctx(), ok, errs, reqs.len() as u32,
                                                      reqs.as_ptr() as *const sys::PeekReq, outs.as_ptr(),
                                                      res.as_mut_ptr()))?;
    }
    Ok(res)
}

impl Drop for GpuPeek {
    fn drop(&mut self) { unsafe { sys::mzgpu_peek_plan_free(self.h) } }
}
