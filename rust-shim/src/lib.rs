//! `mz_compute::gpu` — Rust binding of libmzgpu.so.  UNCOMPILED: see ../README.md.
//!
//! Type aliases in the style of src/compute/src/typedefs.rs:46-126: a dataflow whose arrangement
//! keys/values are fixed-width integer columns instantiates `mz_arrange_core::<_, _, GpuBatcher,
//! GpuBuilder, GpuSpine>` (src/compute/src/extensions/arrange.rs:86-119 is generic over exactly
//! these three parameters).
pub mod batch;
pub mod batcher;
pub mod builder;
pub mod column;
pub mod correction;
pub mod delta_join;
pub mod exchange;
pub mod linear_join;
pub mod mfp;
pub mod peek;
pub mod flat_map;
pub mod reduce;
pub mod sys;
pub mod trace;

pub type GpuKeyValBatcher = batcher::GpuBatcher;
pub type GpuKeyValBuilder = builder::GpuBuilder;
pub type GpuKeyValSpine = trace::GpuSpine;

thread_local! {
    /// One context per timely worker thread (created in Worker::run, src/compute/src/server.rs:350).
    static CTX: std::cell::Cell<*mut sys::Ctx> = std::cell::Cell::new(std::ptr::null_mut());
}
pub fn init_worker(device: i32, worker_index: i32, peers: i32) {
    let mut c = std::ptr::null_mut();
    let st = unsafe { sys::mzgpu_ctx_create(device, worker_index, peers, &mut c) };
    assert_eq!(st, sys::OK, "mzgpu_ctx_create failed");
    CTX.with(|x| x.set(c));
}
pub(crate) fn worker_ctx() -> *mut sys::Ctx { CTX.with(|x| x.get()) }
