//! Delta-join paths over device arrangements.  UNCOMPILED: see ../README.md.
//!
//! `render_delta_join` (src/compute/src/render/join/delta_join.rs:50-311) renders, per source
//! relation, a *path*: `build_update_stream` over the source arrangement's new batch (:312-377),
//! then one `half_join` per other relation (:379-454, `dogs3::half_join` with the `le` / `lt`
//! comparison chosen by relation order, :246-271) with a `JoinClosure` between the stages, and the
//! concatenation of all paths' results (:302-308).  Here the half joins of one stage — independent
//! operators activated by the same frontier advance — are ONE launch: a *chain* is the set of
//! requests appending to one output buffer (the last stage: every path appends to the result
//! collection), chains run side by side.
use super::sys::{self, Closure};
use super::worker_ctx;

/// One stage of one path: probe `trace` with `stream`, keep matches at times `<=` / `<` the
/// stream row's time, apply `closure`, append to `out`.
pub struct HalfJoin<'a> {
    pub stream: *mut sys::Buf,
    pub trace: *mut sys::Spine,
    pub less_equal: bool,
    pub closure: Option<&'a Closure>,
    pub out: *mut sys::Buf,
}

/// The stage-s half joins of all active paths (include/mzgpu.h: `mzgpu_half_join_many`).
pub fn half_join_stage(reqs: &[HalfJoin<'_>]) -> Result<(), (i32, String)> {
    let streams: Vec<_> = reqs.iter().map(|r| r.stream).collect();
    let traces: Vec<_> = reqs.iter().map(|r| r.trace).collect();
    let cmps: Vec<_> = reqs.iter().map(|r| if r.less_equal { sys::HALFJOIN_LE } else { sys::HALFJOIN_LT }).collect();
    let cls: Vec<*const Closure> = reqs.iter().map(|r| r.closure.map_or(std::ptr::null(), |c| c as *const _)).collect();
    let outs: Vec<_> = reqs.iter().map(|r| r.out).collect();
    unsafe {
        sys::check(worker_ctx(), sys::mzgpu_half_join_many(worker_ctx(), reqs.len() as u32, streams.as_ptr(), traces.as_ptr(),
                                                           cmps.as_ptr(), cls.as_ptr(), outs.as_ptr()))
    }
}

/// `build_update_stream` fused into the first half join of every path (one worker: the stream
/// never exists as a collection of its own).  `as_of_skip[j]`: the time whose updates path j must
/// not see (only the first relation's path sees the updates at `as_of`, delta_join.rs:330-345),
/// or `sys::FRONTIER_EMPTY`.
pub fn first_stage(batches: &[*mut sys::Batch], initial: &[*const Closure], as_of_skip: &[u64], traces: &[*mut sys::Spine],
                   less_equal: &[bool], closures: &[*const Closure], outs: &[*mut sys::Buf]) -> Result<(), (i32, String)> {
    let cmps: Vec<_> = less_equal.iter().map(|&le| if le { sys::HALFJOIN_LE } else { sys::HALFJOIN_LT }).collect();
    unsafe {
        sys::check(worker_ctx(), sys::mzgpu_delta_first_stage_many(worker_ctx(), batches.len() as u32, batches.as_ptr(), initial.as_ptr(),
                                                                   as_of_skip.as_ptr(), traces.as_ptr(), cmps.as_ptr(),
                                                                   closures.as_ptr(), outs.as_ptr()))
    }
}

/// The stage-s half joins with `JoinClosure`s outside `mzgpu_closure` (include/mzgpu.h:
/// `mzgpu_half_join_many_mfp`): `closures[j]` from `mzgpu_join_closure_new`, the error rows of every
/// request appended to `errs` (R32, consolidated), the input of the error collection.
pub fn half_join_stage_mfp(streams: &[*mut sys::Buf], traces: &[*mut sys::Spine], less_equal: &[bool],
                           closures: &[*const sys::JoinClosure], outs: &[*mut sys::Buf], errs: *mut sys::Buf)
                           -> Result<(), (i32, String)> {
    let cmps: Vec<_> = less_equal.iter().map(|&le| if le { sys::HALFJOIN_LE } else { sys::HALFJOIN_LT }).collect();
    unsafe {
        sys::check(worker_ctx(), sys::mzgpu_half_join_many_mfp(worker_ctx(), streams.len() as u32, streams.as_ptr(),
                                                               traces.as_ptr(), cmps.as_ptr(), closures.as_ptr(),
                                                               outs.as_ptr(), errs))
    }
}
