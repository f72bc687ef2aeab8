// host.cu — the C ABI of libmzgpu (include/mzgpu.h): contexts, row buffers,
// batcher, batches, the fueled spine, join_core / half_join / reduce operator
// state, and the NCCL exchange.  Host-side bookkeeping only; every per-row
// operation is a CUDA kernel from the sibling .cu files.  There is no CPU
// fallback: without a CUDA device every entry point fails with MZGPU_E_CUDA.
#include <dlfcn.h>

#include <algorithm>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <new>

#include "common.cuh"

// ====================================================================== ctx
static void side_outputs_joined(mzgpu_ctx* ctx);  // (defined with the batch type)
extern "C" int32_t mzgpu_ctx_create(int32_t device, int32_t worker_index, int32_t peers,
                                    mzgpu_ctx** out) {
  if (out == nullptr || peers < 1 || worker_index < 0 || worker_index >= peers) return MZGPU_E_INVALID;
  *out = nullptr;
  mzgpu_ctx* ctx = new (std::nothrow) mzgpu_ctx();
  if (ctx == nullptr) return MZGPU_E_INVALID;
  memset(&ctx->stats, 0, sizeof(ctx->stats));
  ctx->device = device;
  ctx->worker = worker_index;
  ctx->peers = peers;
  *out = ctx;  // returned even on failure so the caller can read mzgpu_last_error
  MZ_CUDA(ctx, cudaSetDevice(device));
  cudaDeviceProp prop;
  MZ_CUDA(ctx, cudaGetDeviceProperties(&prop, device));
  ctx->num_sms = prop.multiProcessorCount;
  MZ_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  MZ_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev, cudaEventDisableTiming));
  if (const char* e = getenv("MZGPU_BLOCKING_SYNC"))
    if (atoi(e) != 0) MZ_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_block, cudaEventDisableTiming | cudaEventBlockingSync));
  MZ_CUDA(ctx, cudaMallocHost((void**)&ctx->h_scratch, 128 * 8));
  MZ_CUDA(ctx, cudaMalloc((void**)&ctx->d_scratch, 128 * 8));
  MZ_CUDA(ctx, cudaMallocHost((void**)&ctx->h_big, 4096));
  // device-resident counters, look-back state, tile tickets, fused control blocks
  MZ_CUDA(ctx, cudaMalloc((void**)&ctx->d_cnt, (size_t)MZ_CNT_BLOCKS * 32));
  MZ_CUDA(ctx, cudaMallocHost((void**)&ctx->h_cnt, (size_t)MZ_CNT_BLOCKS * 32));
  MZ_CUDA(ctx, cudaMalloc((void**)&ctx->d_lb, (size_t)MZ_LB_TILES * 8));
  MZ_CUDA(ctx, cudaMemset(ctx->d_lb, 0, (size_t)MZ_LB_TILES * 8));
  MZ_CUDA(ctx, cudaMalloc((void**)&ctx->d_tickets, (size_t)MZ_TICKETS * 4));
  MZ_CUDA(ctx, cudaMemset(ctx->d_tickets, 0, (size_t)MZ_TICKETS * 4));
  MZ_CUDA(ctx, cudaMalloc((void**)&ctx->d_lb_side, (size_t)MZ_LB_TILES * 8));
  MZ_CUDA(ctx, cudaMemset(ctx->d_lb_side, 0, (size_t)MZ_LB_TILES * 8));
  MZ_CUDA(ctx, cudaMalloc((void**)&ctx->d_tickets_side, (size_t)MZ_TICKETS * 4));
  MZ_CUDA(ctx, cudaMemset(ctx->d_tickets_side, 0, (size_t)MZ_TICKETS * 4));
  MZ_CUDA(ctx, cudaMalloc((void**)&ctx->d_status, 16));
  MZ_CUDA(ctx, cudaMemset(ctx->d_status, 0, 16));
  for (int i = 0; i < 4; ++i) {
    MZ_CUDA(ctx, cudaMalloc(&ctx->d_fused_ctl[i], mz_fused_ctl_bytes()));
    MZ_CUDA(ctx, cudaMemset(ctx->d_fused_ctl[i], 0, mz_fused_ctl_bytes()));
  }
  if (const char* e = getenv("MZGPU_MID_BLOCK_MB")) ctx->mid_block = (size_t)strtoull(e, nullptr, 10) << 20;
  for (int i = 0; i < 16; ++i) {
    MZ_CUDA(ctx, cudaMalloc(&ctx->d_fused_ctl_many[i], mz_fused_ctl_bytes()));
    MZ_CUDA(ctx, cudaMemset(ctx->d_fused_ctl_many[i], 0, mz_fused_ctl_bytes()));
  }
  ctx->main_stream = ctx->stream;
  MZ_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->side_stream, cudaStreamNonBlocking));
  MZ_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
  MZ_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_side, cudaEventDisableTiming));
  // keep freed blocks cached in the stream-ordered pool
  cudaMemPool_t pool;
  MZ_CUDA(ctx, cudaDeviceGetDefaultMemPool(&pool, device));
  uint64_t thresh = UINT64_MAX;
  MZ_CUDA(ctx, cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
  // Pre-size the pool: operator scratch is sized by upper bounds (hundreds of MB per
  // update batch, released in stream order right away) and growing the pool on the
  // hot path costs milliseconds.  One reservation up front; MZGPU_POOL_MB overrides.
  {
    size_t free_b = 0, total_b = 0;
    MZ_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    size_t want = (size_t)40 << 30;  // (blocks parked in the library's own caches, DevMem, are not free memory of the pool)
    if (const char* e = getenv("MZGPU_POOL_MB")) want = (size_t)strtoull(e, nullptr, 10) << 20;
    if (want > free_b / 2) want = free_b / 2;
    if (want >= ((size_t)1 << 20)) {
      void* p = nullptr;
      MZ_CUDA(ctx, cudaMallocAsync(&p, want, ctx->stream));
      MZ_CUDA(ctx, cudaFreeAsync(p, ctx->stream));
      MZ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
  }
  return MZGPU_OK;
}

extern "C" void mzgpu_ctx_destroy(mzgpu_ctx* ctx) {
  if (ctx == nullptr) return;
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->side_stream) cudaStreamSynchronize(ctx->side_stream);
  ctx->stream = ctx->main_stream ? ctx->main_stream : ctx->stream;
  ctx->joined_seq = ctx->side_seq;
  side_outputs_joined(ctx);  // merges that were never joined: let go of their inputs
  if (ctx->nccl_comm && ctx->nccl_lib) {
    typedef int (*destroy_t)(void*);
    destroy_t f = (destroy_t)dlsym(ctx->nccl_lib, "ncclCommDestroy");
    if (f) f(ctx->nccl_comm);
  }
  if (ctx->h_scratch) cudaFreeHost(ctx->h_scratch);
  if (ctx->h_big) cudaFreeHost(ctx->h_big);
  if (ctx->h_cnt) cudaFreeHost(ctx->h_cnt);
  if (ctx->d_cnt) cudaFree(ctx->d_cnt);
  if (ctx->d_lb) cudaFree(ctx->d_lb);
  if (ctx->d_tickets) cudaFree(ctx->d_tickets);
  if (ctx->d_lb_side) cudaFree(ctx->d_lb_side);
  if (ctx->d_tickets_side) cudaFree(ctx->d_tickets_side);
  if (ctx->d_status) cudaFree(ctx->d_status);
  if (ctx->d_dbg) cudaFree(ctx->d_dbg);
  for (int i = 0; i < 4; ++i)
    if (ctx->d_fused_ctl[i]) cudaFree(ctx->d_fused_ctl[i]);
  for (int i = 0; i < 16; ++i)
    if (ctx->d_fused_ctl_many[i]) cudaFree(ctx->d_fused_ctl_many[i]);
  mz_fused_deferred_free(ctx);
  for (auto& b : ctx->big_cache) cudaFree(b.p);
  for (auto& b : ctx->mid_cache) cudaFree(b.p);
  ctx->big_cache.clear();
  for (int p = 0; p < 16; ++p)
    if (ctx->p2p_peer_ipc[p] && ctx->p2p_peer[p]) cudaIpcCloseMemHandle(ctx->p2p_peer[p]);
  if (ctx->p2p_local) cudaFree(ctx->p2p_local);
  if (ctx->p2p_cursors) cudaFree(ctx->p2p_cursors);
  if (ctx->side_stream) {
    cudaStreamSynchronize(ctx->side_stream);
    cudaStreamDestroy(ctx->side_stream);
  }
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_side) cudaEventDestroy(ctx->ev_side);
  ctx->stream = ctx->main_stream;
  if (ctx->d_scratch) cudaFree(ctx->d_scratch);
  if (ctx->ev) cudaEventDestroy(ctx->ev);
  if (ctx->ev_block) cudaEventDestroy(ctx->ev_block);
  for (auto& r : ctx->prof) {
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  for (auto e : ctx->ev_pool) cudaEventDestroy(e);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

extern "C" const char* mzgpu_last_error(mzgpu_ctx* ctx) {
  return ctx ? ctx->last_error.c_str() : "null context";
}

// ------------------------------------------------ device-resident counters
int mz_cnt_alloc(mzgpu_ctx* ctx) {
  if (!ctx->cnt_free.empty()) {
    int b = ctx->cnt_free.back();
    ctx->cnt_free.pop_back();
    return b;
  }
  if (ctx->cnt_high < MZ_CNT_BLOCKS) return ctx->cnt_high++;
  return -1;
}
void mz_cnt_free(mzgpu_ctx* ctx, int blk) {
  if (ctx == nullptr || blk < 0) return;
  // A block may still be written by a kernel in flight.  On one stream that is harmless (its
  // next producer is queued behind that kernel); while side-stream work is outstanding the
  // next producer could run on the other stream, so the block is parked until the join.
  // The same holds while prepared-but-unlaunched (deferred) jobs exist: such a job may read
  // this block (an input length captured as a device pointer), and the block's next producer
  // would be enqueued AHEAD of the deferred launch -- parked until the flush.
  if (ctx->stream != ctx->main_stream || ctx->joined_seq != ctx->side_seq || ctx->deferred_unlaunched > 0)
    ctx->cnt_parked.push_back(blk);
  else
    ctx->cnt_free.push_back(blk);
}
// parked blocks become reusable once nothing unlaunched or unjoined can touch them
void mz_cnt_unpark(mzgpu_ctx* ctx) {
  if (ctx->stream != ctx->main_stream || ctx->joined_seq != ctx->side_seq || ctx->deferred_unlaunched > 0) return;
  for (int b : ctx->cnt_parked) ctx->cnt_free.push_back(b);
  ctx->cnt_parked.clear();
}
// One copy of the whole arena (a few KB) + one wait: every count produced by a
// kernel enqueued before this call becomes readable on the host.
// the main stream waits for every merge issued on the side stream so far
static void batch_release_internal(struct mzgpu_batch* b);
static void side_outputs_joined(mzgpu_ctx* ctx);  // (after the batch type is complete)
static int32_t mz_join_side(mzgpu_ctx* ctx) {
  if (ctx->joined_seq == ctx->side_seq) return MZGPU_OK;
  if (ctx->stream == ctx->main_stream) {
    MZ_CUDA(ctx, cudaStreamWaitEvent(ctx->main_stream, ctx->ev_side, 0));
    mz_mid_joined(ctx);
    ctx->joined_seq = ctx->side_seq;
    side_outputs_joined(ctx);
    mz_cnt_unpark(ctx);
  }
  return MZGPU_OK;
}
static int32_t mz_flush_deferred(mzgpu_ctx* ctx);
int32_t mz_resolve_counters(mzgpu_ctx* ctx) {
  MZ_CHECK_CTX(ctx);
  // counters of deferred jobs count as written: their launch must precede the copy
  MZ_TRY(mz_flush_deferred(ctx));
  // Counts written on the side stream are NOT waited for: the counter blocks of a merge in flight
  // there carry seq = ~0 until the main stream joins it (mz_join_side), so this copy never passes
  // for their value, and the operators of a timestamp keep running beside the merges it triggered.
  if (ctx->stream != ctx->main_stream) MZ_CUDA(ctx, cudaStreamSynchronize(ctx->main_stream));
  const size_t bytes = (size_t)ctx->cnt_high * 32;
  if (bytes) MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_cnt, ctx->d_cnt, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 40, ctx->d_status, 16, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += bytes + 16;
  ctx->resolved_seq = ctx->op_seq;
  ctx->n_resolves++;
  if (ctx->h_scratch[40] != 0) {
    MZ_SET_ERR(ctx, "internal: a bounded operator output overflowed its capacity (%llu rows required)",
               (unsigned long long)ctx->h_scratch[40]);
    ctx->sticky = true;
    ctx->sticky_code = MZGPU_E_CAPACITY;
    return MZGPU_E_CAPACITY;
  }
  if (ctx->h_scratch[41] != 0) {
    MZ_SET_ERR(ctx, "MIN/MAX reduce: a key has more than 32 distinct live values (bucketed reduction tree "
                    "not implemented)");
    ctx->sticky = true;
    ctx->sticky_code = MZGPU_E_UNSUPPORTED;
    return MZGPU_E_UNSUPPORTED;
  }
  return MZGPU_OK;
}
int32_t mz_lookback_begin(mzgpu_ctx* ctx, u64 max_tiles, LookBack* lb) {
  return mz_lookback_begin_at(ctx, 0, max_tiles, lb);
}
int32_t mz_lookback_begin_at(mzgpu_ctx* ctx, u64 at, u64 max_tiles, LookBack* lb) {
  if (at + max_tiles > MZ_LB_TILES) {
    MZ_SET_ERR(ctx, "single-pass kernel: %llu tiles exceed the look-back state",
               (unsigned long long)(at + max_tiles));
    return MZGPU_E_UNSUPPORTED;
  }
  const bool side = ctx->side_stream != nullptr && ctx->stream == ctx->side_stream;
  ctx->lb_epoch = (ctx->lb_epoch + 1) & 0xfffffu;
  if (ctx->lb_epoch == 0) {  // tag space wrapped (once per million launches): clear both state arrays
    if (ctx->side_stream != nullptr) MZ_CUDA(ctx, cudaStreamSynchronize(side ? ctx->main_stream : ctx->side_stream));
    MZ_CUDA(ctx, cudaMemsetAsync(ctx->d_lb, 0, (size_t)MZ_LB_TILES * 8, ctx->stream));
    MZ_CUDA(ctx, cudaMemsetAsync(ctx->d_lb_side, 0, (size_t)MZ_LB_TILES * 8, ctx->stream));
    MZ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->lb_epoch = 1;
  }
  u32& next = side ? ctx->ticket_next_side : ctx->ticket_next;
  u32* tickets = side ? ctx->d_tickets_side : ctx->d_tickets;
  if (next == MZ_TICKETS) {
    MZ_CUDA(ctx, cudaMemsetAsync(tickets, 0, (size_t)MZ_TICKETS * 4, ctx->stream));
    next = 0;
  }
  lb->state = (side ? ctx->d_lb_side : ctx->d_lb) + at;
  lb->ticket = tickets + next++;
  lb->epoch = ctx->lb_epoch;
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_ctx_sync(mzgpu_ctx* ctx) {
  MZ_CHECK_CTX(ctx);
  return mz_resolve_counters(ctx);
}

extern "C" int32_t mzgpu_ctx_stats(mzgpu_ctx* ctx, mzgpu_stats* out) {
  if (ctx == nullptr || out == nullptr) return MZGPU_E_INVALID;
  if (getenv("MZGPU_DEBUG"))
    fprintf(stderr,
            "[mzgpu] allocs %llu (%.1f MB, %.3f ms host)  syncs %llu (%.3f ms waiting)  launches %llu  counter blocks %d"
            " in use (high water %d)  big blocks: %llu reused, %llu new, %.1f MB parked  mid blocks: %llu reused, %llu new,"
            " %.1f MB parked\n",
            (unsigned long long)ctx->n_alloc, ctx->bytes_alloc / 1e6, ctx->ns_alloc / 1e6,
            (unsigned long long)ctx->stats.host_syncs, ctx->ns_sync / 1e6,
            (unsigned long long)ctx->stats.kernel_launches, ctx->cnt_high - (int)ctx->cnt_free.size(), ctx->cnt_high,
            (unsigned long long)ctx->big_hits, (unsigned long long)ctx->big_misses, ctx->big_cached_bytes / 1e6,
            (unsigned long long)ctx->mid_hits, (unsigned long long)ctx->mid_misses, ctx->mid_cached_bytes / 1e6);
  *out = ctx->stats;
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_ctx_host_times(mzgpu_ctx* ctx, uint64_t out[4]) {
  if (ctx == nullptr || out == nullptr) return MZGPU_E_INVALID;
  out[0] = ctx->ns_sync;
  out[1] = ctx->ns_alloc;
  out[2] = ctx->n_alloc;
  out[3] = ctx->bytes_alloc;
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_profile_enable(mzgpu_ctx* ctx, int32_t on) {
  MZ_CHECK_CTX(ctx);
  ctx->profile = on != 0;
  if (on && ctx->d_dbg == nullptr) MZ_CUDA(ctx, cudaMalloc((void**)&ctx->d_dbg, (size_t)MZ_DBG_RECORDS * 32 * 8));
  if (on) ctx->dbg_next = 0;
  return MZGPU_OK;
}
// Phase stamps of the fused kernel's launches since profiling was enabled:
// 32 words per launch ([0..9] globaltimer ns at phase boundaries, [16] rows,
// [17] radix rounds, [18] bits per round, [19] CTAs used).  Returns the count.
extern "C" int32_t mzgpu_profile_fused_phases(mzgpu_ctx* ctx, uint64_t* out, uint32_t cap_records, uint32_t* n) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || n == nullptr) return MZGPU_E_INVALID;
  MZ_SYNC(ctx);
  uint32_t m = ctx->dbg_next < cap_records ? ctx->dbg_next : cap_records;
  if (m) MZ_CUDA(ctx, cudaMemcpy(out, ctx->d_dbg, (size_t)m * 32 * 8, cudaMemcpyDeviceToHost));
  *n = m;
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_profile_report(mzgpu_ctx* ctx, char* buf, uint64_t cap) {
  MZ_CHECK_CTX(ctx);
  if (buf == nullptr || cap == 0) return MZGPU_E_INVALID;
  MZ_SYNC(ctx);
  struct Agg {
    std::string name;
    u64 launches = 0, bytes = 0;
    double ms = 0;
  };
  std::vector<Agg> aggs;
  for (auto& r : ctx->prof) {
    float ms = 0;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    Agg* a = nullptr;
    for (auto& x : aggs)
      if (x.name == r.name) a = &x;
    if (a == nullptr) {
      aggs.push_back(Agg());
      a = &aggs.back();
      a->name = r.name;
    }
    a->launches++;
    a->bytes += r.bytes;
    a->ms += ms;
    ctx->ev_pool.push_back(r.e0);
    ctx->ev_pool.push_back(r.e1);
  }
  ctx->prof.clear();
  // the fused kernel leaves its actual row count in its debug record
  if (ctx->d_dbg != nullptr && ctx->dbg_next > 0) {
    std::vector<u64> rec((size_t)ctx->dbg_next * 32);
    if (cudaMemcpy(rec.data(), ctx->d_dbg, rec.size() * 8, cudaMemcpyDeviceToHost) == cudaSuccess) {
      u64 bytes = 0;
      for (u32 i = 0; i < ctx->dbg_next; ++i) bytes += rec[(size_t)i * 32 + 16] * rec[(size_t)i * 32 + 20] * 4;
      for (auto& x : aggs)
        // (one record per job: a multi-job launch leaves several)
        if (x.name == "k_fused_consolidate" && x.launches <= ctx->dbg_next) x.bytes = bytes;
    }
    ctx->dbg_next = 0;
  }
  std::string out;
  for (auto& a : aggs) {
    char line[384];
    std::string nm = a.name;
    for (auto& ch : nm)
      if (ch == ' ') ch = '_';
    snprintf(line, sizeof(line), "%s %llu %.6f %llu\n", nm.c_str(), (unsigned long long)a.launches, a.ms,
             (unsigned long long)a.bytes);
    out += line;
  }
  if (out.size() + 1 > cap) return MZGPU_E_CAPACITY;
  memcpy(buf, out.c_str(), out.size() + 1);
  return MZGPU_OK;
}

extern "C" void* mzgpu_ctx_stream(mzgpu_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

// ------------------------------------------------------------- transfers
static int32_t copy_in(mzgpu_ctx* ctx, void* d_dst, const void* src, size_t bytes, int32_t mem) {
  if (bytes == 0) return MZGPU_OK;
  if (mem == MZGPU_MEM_HOST) {
    MZ_CUDA(ctx, cudaMemcpyAsync(d_dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    ctx->stats.h2d_bytes += bytes;
  } else {
    MZ_CUDA(ctx, cudaMemcpyAsync(d_dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  return MZGPU_OK;
}
static int32_t copy_out(mzgpu_ctx* ctx, void* dst, const void* d_src, size_t bytes, int32_t mem) {
  if (bytes == 0) return MZGPU_OK;
  if (mem == MZGPU_MEM_HOST) {
    MZ_CUDA(ctx, cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    MZ_SYNC(ctx);
    ctx->stats.d2h_bytes += bytes;
  } else {
    MZ_CUDA(ctx, cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  return MZGPU_OK;
}

// The rows of a host-form entry point (n rows of in_rb bytes) counted into rows_in and, when they are in host
// memory, uploaded into `in`; *d_rows is where the operator reads them.
static int32_t entry_rows_in(mzgpu_ctx* ctx, const void* rows, uint64_t n, int32_t mem, uint32_t in_rb, DevMem* in,
                             const u64** d_rows) {
  ctx->stats.rows_in += n;
  *d_rows = (const u64*)rows;
  if (mem == MZGPU_MEM_HOST && n) {
    MZ_TRY(in->alloc(ctx, n * in_rb));
    MZ_TRY(copy_in(ctx, in->p, rows, n * in_rb, mem));
    *d_rows = in->as<u64>();
  }
  return MZGPU_OK;
}

// Closure descriptors come from the caller: everything the device code indexes or shifts by is
// checked here, once, at plan time (include/mzgpu.h: richer plans are MZGPU_E_UNSUPPORTED, malformed
// descriptors MZGPU_E_INVALID; nothing undefined reaches a kernel).
static int32_t validate_field(mzgpu_ctx* ctx, const mzgpu_field& f, bool uses_dst) {
  if (f.src > MZGPU_SRC_VAL2 || f.shift >= 64 || f.bits < 1 || f.bits > 64 || (uses_dst && f.dst_shift >= 64)) {
    MZ_SET_ERR(ctx, "closure: bad field {src=%u shift=%u bits=%u dst_shift=%u}", f.src, f.shift, f.bits, f.dst_shift);
    return MZGPU_E_INVALID;
  }
  return MZGPU_OK;
}
static int32_t validate_closure(mzgpu_ctx* ctx, const mzgpu_closure* c) {
  if (c == nullptr) return MZGPU_OK;
  if (c->n_key_fields > MZGPU_MAX_FIELDS || c->n_val_fields > MZGPU_MAX_FIELDS || c->n_filters > MZGPU_MAX_FILTERS) {
    MZ_SET_ERR(ctx, "closure: %u key fields / %u value fields / %u filters exceed the descriptor (%d / %d / %d)",
               c->n_key_fields, c->n_val_fields, c->n_filters, MZGPU_MAX_FIELDS, MZGPU_MAX_FIELDS, MZGPU_MAX_FILTERS);
    return MZGPU_E_UNSUPPORTED;
  }
  if (c->expr_kind != MZGPU_EXPR_NONE && c->expr_kind != MZGPU_EXPR_MUL_CONST_MINUS) {
    MZ_SET_ERR(ctx, "closure: unknown expression kind %u", c->expr_kind);
    return MZGPU_E_UNSUPPORTED;
  }
  for (uint32_t i = 0; i < c->n_key_fields; ++i) MZ_TRY(validate_field(ctx, c->key_fields[i], true));
  if (c->expr_kind == MZGPU_EXPR_MUL_CONST_MINUS) {
    MZ_TRY(validate_field(ctx, c->expr_a, false));
    MZ_TRY(validate_field(ctx, c->expr_b, false));
  } else {
    for (uint32_t i = 0; i < c->n_val_fields; ++i) MZ_TRY(validate_field(ctx, c->val_fields[i], true));
  }
  for (uint32_t i = 0; i < c->n_filters; ++i) {
    MZ_TRY(validate_field(ctx, c->filters[i].field, false));
    if (c->filters[i].op > MZGPU_CMP_GE) {
      MZ_SET_ERR(ctx, "closure: unknown comparison %u", c->filters[i].op);
      return MZGPU_E_UNSUPPORTED;
    }
  }
  return MZGPU_OK;
}

// arrangement rows: every sorted-batch width but the reduce's 64-byte output rows, i.e. R32, the
// accumulable rows of every lane class (RACC = class 1) and the monotonic reduce's rows
static bool arrangement_row_bytes(uint32_t rb) { return rb != 64 && BatchWidths::has((int)rb); }
// buffer rows: every RowT width, and the output rows of the lanes and monotonic reduces (they have no RowT)
static bool valid_row_bytes(uint32_t rb) {
  return RowWidths::has((int)rb) || rb == 96 || rb == 144 || rb == 240 || rb == 56 || rb == 88;
}

// ------------------------------------------------------ device-side append
// dst[base ...] = src[0 .. n), new length left in *out_len; every size may live
// in device memory.
namespace {
__global__ void __launch_bounds__(256) k_append_rows(const u64* __restrict__ src, const DLen dn, int nw,
                                                     u64* __restrict__ dst, const DLen dbase, u64 cap_rows,
                                                     u64* __restrict__ out_len, u64* __restrict__ status) {
  const u64 n = dlen_get(dn), base = dlen_get(dbase);
  const u64 gtid = (u64)blockIdx.x * 256 + threadIdx.x, stride = (u64)gridDim.x * 256;
  u64 m = n;
  if (base + n > cap_rows) {
    if (gtid == 0) atomicMax((unsigned long long*)status, (unsigned long long)(base + n));
    m = cap_rows > base ? cap_rows - base : 0;
  }
  const u64 words = m * (u64)nw;
  u64* d = dst + base * (u64)nw;
  for (u64 i = gtid; i < words; i += stride) d[i] = src[i];
  if (gtid == 0) *out_len = base + n;
}
}  // namespace

static int32_t append_dev(mzgpu_ctx* ctx, const void* src, DLen n, u64 n_ub, int rb, void* dst, DLen base,
                          u64 cap_rows, u64* out_len) {
  u64 grid = (n_ub * (u64)(rb / 8) + 1023) / 1024;
  const u64 maxg = (u64)ctx->num_sms * 8;
  if (grid > maxg) grid = maxg;
  if (grid == 0) grid = 1;
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * rb * 2 : 0);
  MZ_LAUNCH(ctx, k_append_rows, (unsigned)grid, 256, 0, (const u64*)src, n, rb / 8, (u64*)dst, base, cap_rows,
            out_len, ctx->d_status);
  return MZGPU_OK;
}

// ====================================================================== buf
struct mzgpu_buf {
  mzgpu_ctx* ctx;
  uint32_t rb;
  DevMem mem;
  u64 cap = 0;
  Lazy4 len;     // the row count is word `word` of the block while it is pending
  int word = 0;
  u64 ub = 0;    // host upper bound on the row count (exact when len.known)
};

static DLen buf_dlen(const mzgpu_buf* b) { return dlen_of(b->len, b->word); }
static void buf_set_len(mzgpu_buf* b, u64 n) {
  b->len.set(b->ctx, n);
  b->word = 0;
  b->ub = n;
}
static int32_t buf_resolve(mzgpu_buf* b) {
  if (b->len.known) return MZGPU_OK;
  MZ_TRY(b->len.resolve());
  buf_set_len(b, b->len.v[b->word]);
  return MZGPU_OK;
}
// An operator is about to append a device-counted number of rows: where it
// reads the current length and where it leaves the new one (never the same word).
struct Append {
  DLen base;
  u64* out_len;
  int new_word;
};
static int32_t buf_begin_append(mzgpu_buf* b, Append* a) {
  if (b->len.known) {
    a->base = dlen_imm(b->len.v[b->word]);
    MZ_TRY(b->len.make_pending(b->ctx));
    a->out_len = b->len.dptr();
    a->new_word = 0;
  } else {
    a->base.p = b->len.dptr() + b->word;
    a->base.imm = 0;
    a->out_len = b->len.dptr() + (b->word ^ 1);
    a->new_word = b->word ^ 1;
  }
  return MZGPU_OK;
}
static void buf_end_append(mzgpu_buf* b, const Append& a, u64 added_ub) {
  b->word = a.new_word;
  b->len.mark_written();
  b->ub += added_ub;
}

static int32_t buf_reserve(mzgpu_buf* b, u64 n, bool keep) {
  if (n <= b->cap) return MZGPU_OK;
  u64 ncap = std::max<u64>(n, b->cap * 2);
  DevMem m;
  MZ_TRY(m.alloc(b->ctx, ncap * b->rb));
  if (keep && b->ub) MZ_TRY(copy_in(b->ctx, m.p, b->mem.p, b->ub * b->rb, MZGPU_MEM_DEVICE));
  b->mem = std::move(m);
  b->cap = ncap;
  return MZGPU_OK;
}
// take ownership of a device array as the buffer contents
static void buf_adopt(mzgpu_buf* b, DevMem&& m, u64 len) {
  b->cap = m.bytes / b->rb;
  b->mem = std::move(m);
  buf_set_len(b, len);
}
// append n device rows; n may be device resident
static int32_t buf_append_dev(mzgpu_buf* b, const void* d_rows, DLen n, u64 n_ub) {
  if (n_ub == 0) return MZGPU_OK;
  MZ_TRY(buf_reserve(b, b->ub + n_ub, true));
  if (b->len.known && n.p == nullptr) {
    MZ_TRY(copy_in(b->ctx, (char*)b->mem.p + b->ub * b->rb, d_rows, n.imm * b->rb, MZGPU_MEM_DEVICE));
    buf_set_len(b, b->ub + n.imm);
    return MZGPU_OK;
  }
  Append a;
  MZ_TRY(buf_begin_append(b, &a));
  MZ_TRY(append_dev(b->ctx, d_rows, n, n_ub, b->rb, b->mem.p, a.base, b->cap, a.out_len));
  buf_end_append(b, a, n_ub);
  return MZGPU_OK;
}

// append src's rows where the CALLER bounds their number (tighter than the library's own bound):
// the destination grows by at most `max_rows`; more rows than that are detected on the device
// (reported as MZGPU_E_CAPACITY at the next read-back, nothing is written past the capacity)
extern "C" int32_t mzgpu_buf_append_buf_at_most(mzgpu_buf* dst, mzgpu_buf* src, uint64_t max_rows) {
  if (dst == nullptr || src == nullptr || dst == src || dst->rb != src->rb) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(dst->ctx);
  const u64 n_ub = std::min<u64>(src->ub, max_rows);
  if (n_ub == 0) return MZGPU_OK;
  mzgpu_ctx* ctx = dst->ctx;
  MZ_TRY(buf_reserve(dst, dst->ub + n_ub, true));
  if (dst->len.known && src->len.known) {
    if (src->len.v[src->word] > max_rows) {
      MZ_SET_ERR(ctx, "buf_append_buf_at_most: %llu rows exceed the caller's bound %llu",
                 (unsigned long long)src->len.v[src->word], (unsigned long long)max_rows);
      return MZGPU_E_CAPACITY;
    }
    return buf_append_dev(dst, src->mem.p, buf_dlen(src), n_ub);
  }
  Append a;
  MZ_TRY(buf_begin_append(dst, &a));
  // capacity as seen by the kernel = what this append may fill at most
  MZ_TRY(append_dev(ctx, src->mem.p, buf_dlen(src), src->ub, dst->rb, dst->mem.p, a.base, dst->ub + n_ub, a.out_len));
  buf_end_append(dst, a, n_ub);
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_buf_new(mzgpu_ctx* ctx, uint32_t row_bytes, mzgpu_buf** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || !valid_row_bytes(row_bytes)) return MZGPU_E_INVALID;
  mzgpu_buf* b = new mzgpu_buf();
  b->ctx = ctx;
  b->rb = row_bytes;
  b->len.set(ctx, 0);
  *out = b;
  return MZGPU_OK;
}
extern "C" void mzgpu_buf_free(mzgpu_buf* b) { delete b; }
extern "C" uint64_t mzgpu_buf_len(const mzgpu_buf* b) {
  if (b == nullptr) return 0;
  if (buf_resolve(const_cast<mzgpu_buf*>(b)) != MZGPU_OK) return 0;
  return b->ub;
}
extern "C" uint32_t mzgpu_buf_row_bytes(const mzgpu_buf* b) { return b ? b->rb : 0; }
extern "C" void* mzgpu_buf_device_ptr(mzgpu_buf* b) { return b ? b->mem.p : nullptr; }
extern "C" int32_t mzgpu_buf_clear(mzgpu_buf* b) {
  if (b == nullptr) return MZGPU_E_INVALID;
  buf_set_len(b, 0);
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_buf_upload(mzgpu_buf* b, const void* rows, uint64_t n, int32_t mem) {
  if (b == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  buf_set_len(b, 0);
  MZ_TRY(buf_reserve(b, n, false));
  MZ_TRY(copy_in(b->ctx, b->mem.p, rows, n * b->rb, mem));
  buf_set_len(b, n);
  b->ctx->stats.rows_in += n;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_buf_append(mzgpu_buf* b, const void* rows, uint64_t n, int32_t mem) {
  if (b == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  b->ctx->stats.rows_in += n;
  if (n == 0) return MZGPU_OK;
  if (mem == MZGPU_MEM_DEVICE) return buf_append_dev(b, rows, dlen_imm(n), n);
  MZ_TRY(buf_resolve(b));  // host rows land at an offset the host must know
  MZ_TRY(buf_reserve(b, b->ub + n, true));
  MZ_TRY(copy_in(b->ctx, (char*)b->mem.p + b->ub * b->rb, rows, n * b->rb, mem));
  buf_set_len(b, b->ub + n);
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_buf_append_buf(mzgpu_buf* dst, mzgpu_buf* src) {
  if (dst == nullptr || src == nullptr || dst == src || dst->rb != src->rb) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(dst->ctx);
  return buf_append_dev(dst, src->mem.p, buf_dlen(src), src->ub);
}
extern "C" int32_t mzgpu_buf_download(mzgpu_buf* b, void* rows, uint64_t cap, int32_t mem,
                                      uint64_t* n_out) {
  if (b == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  MZ_TRY(buf_resolve(b));
  if (n_out) *n_out = b->ub;
  if (cap < b->ub) {
    MZ_SET_ERR(b->ctx, "buf_download: capacity %llu < %llu rows", (unsigned long long)cap,
               (unsigned long long)b->ub);
    return MZGPU_E_CAPACITY;
  }
  MZ_TRY(copy_out(b->ctx, rows, b->mem.p, b->ub * b->rb, mem));
  b->ctx->stats.rows_out += b->ub;
  return MZGPU_OK;
}

// ============================================================ consolidation
// a row count on the host: when it is on the device, every count enqueued so far is read back (one wait)
static int32_t dlen_read(mzgpu_ctx* ctx, DLen n, u64* out) {
  *out = n.imm;
  if (n.p != nullptr) {
    MZ_TRY(mz_resolve_counters(ctx));
    *out = ctx->h_cnt[n.p - ctx->d_cnt];  // the block is part of the arena mirror
  }
  return MZGPU_OK;
}

// rows (device, count possibly device resident) -> consolidated rows; the fused
// kernel for small / medium inputs, the multi-kernel path beyond.
static int32_t consolidate_dev(mzgpu_ctx* ctx, int rb, const void* d_in, DLen n, u64 n_ub, DevMem* out,
                               u64* out_cap, Lazy4* out_len) {
  if (n.p != nullptr && !mz_use_fused(false, n_ub)) {
    // bound too loose to size buffers by: read the count back
    MZ_TRY(dlen_read(ctx, n, &n_ub));
    n = dlen_imm(n_ub);
  }
  if (mz_use_fused(n.p == nullptr, n_ub)) {
    FusedJob job;
    job.rb = rb;
    job.a = d_in;
    job.na = n;
    job.cap = n_ub;
    FusedOut fo;
    MZ_TRY(mz_fused_consolidate(ctx, job, &fo));
    *out = std::move(fo.rows);
    *out_cap = fo.rows_cap;
    *out_len = std::move(fo.st);
    return MZGPU_OK;
  }
  u64 nn = n.imm;
  u64 n_out = 0;
  MZ_TRY(mz_sort_consolidate(ctx, rb, d_in, nn, out, &n_out));
  *out_cap = nn;
  out_len->set(ctx, n_out);
  return MZGPU_OK;
}

// append `n` device rows (count possibly on the device, bound ub) to `dst`, consolidated
static int32_t append_consolidated(mzgpu_ctx* ctx, int rb, const void* d_rows, DLen n, u64 ub, mzgpu_buf* dst) {
  if (ub == 0) return MZGPU_OK;
  DevMem cons;
  u64 cap = 0;
  Lazy4 len;
  MZ_TRY(consolidate_dev(ctx, rb, d_rows, n, ub, &cons, &cap, &len));
  return buf_append_dev(dst, cons.p, dlen_of(len, 0), len.known ? len.v[0] : std::min(cap, ub));
}

static int32_t consolidate_ptr(mzgpu_ctx* ctx, int rb, void* rows, u64 n, int32_t mem, u64* n_out) {
  MZ_CHECK_CTX(ctx);
  if ((rows == nullptr && n) || n_out == nullptr) return MZGPU_E_INVALID;
  *n_out = 0;
  if (n == 0) return MZGPU_OK;
  ctx->stats.rows_in += n;
  DevMem in, out;
  const void* d_in = rows;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(in.alloc(ctx, n * rb));
    MZ_TRY(copy_in(ctx, in.p, rows, n * rb, mem));
    d_in = in.p;
  }
  u64 cap = 0;
  Lazy4 len;
  MZ_TRY(consolidate_dev(ctx, rb, d_in, dlen_imm(n), n, &out, &cap, &len));
  MZ_TRY(len.resolve());
  *n_out = len.v[0];
  MZ_TRY(copy_out(ctx, rows, out.p, *n_out * rb, mem));
  ctx->stats.rows_out += *n_out;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_consolidate_r16(mzgpu_ctx* ctx, mzgpu_r16* rows, uint64_t n, int32_t mem,
                                         uint64_t* n_out) {
  return consolidate_ptr(ctx, 16, rows, n, mem, n_out);
}
extern "C" int32_t mzgpu_consolidate_r32(mzgpu_ctx* ctx, mzgpu_r32* rows, uint64_t n, int32_t mem,
                                         uint64_t* n_out) {
  return consolidate_ptr(ctx, 32, rows, n, mem, n_out);
}
extern "C" int32_t mzgpu_buf_consolidate(mzgpu_buf* b) {
  if (b == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  if (b->ub == 0) return MZGPU_OK;
  DevMem out;
  u64 cap = 0;
  Lazy4 len;
  MZ_TRY(consolidate_dev(b->ctx, b->rb, b->mem.p, buf_dlen(b), b->ub, &out, &cap, &len));
  b->mem = std::move(out);
  b->cap = cap;
  b->ub = len.known ? len.v[0] : b->ub;
  b->len = std::move(len);
  b->word = 0;
  return MZGPU_OK;
}

// ================================================================== batches
struct mzgpu_batch {
  mzgpu_ctx* ctx;
  uint32_t rb;
  DevMem rows;
  u64 rows_cap = 0;
  DevMem table;
  Lazy4 st;        // [0] len, [1] table mask, [2] distinct keys, [3] longest key run (saturating at 1024)
  u64 len_ub = 0;  // host upper bound on len
  mzgpu_desc desc;
  int refs = 1;
  u64 side_seq = 0;  // != 0: produced by merge #side_seq on the side stream
  u64 deferred_seq = 0;  // != 0: produced by deferred job #deferred_seq (launched at the next flush)
  // a merge running on the side stream keeps its inputs: until the main stream has joined that merge,
  // readers (probes) use the inputs in place of this batch -- the reference's readers likewise see a
  // merge's source batches until the merge completes (Spine: in-progress merges keep both batches)
  mzgpu_batch* src1 = nullptr;
  mzgpu_batch* src2 = nullptr;
};
// Launch the deferred merges (one multi-job launch) and let go of their inputs.
static int32_t mz_flush_deferred(mzgpu_ctx* ctx) {
  if (ctx->flushed_seq == ctx->defer_seq) return MZGPU_OK;
  ctx->flushed_seq = ctx->defer_seq;
  const int32_t st = mz_fused_flush(ctx);
  std::vector<mzgpu_batch*> ins;
  ins.swap(ctx->deferred_inputs);
  for (auto* b : ins) batch_release_internal(b);  // freed in stream order, behind the launch
  return st;
}
// before the main stream reads or frees a batch: wait for the merge that produced it
static int32_t batch_ready(mzgpu_batch* b) {
  if (b->deferred_seq > b->ctx->flushed_seq) MZ_TRY(mz_flush_deferred(b->ctx));
  if (b->side_seq > b->ctx->joined_seq) return mz_join_side(b->ctx);
  return MZGPU_OK;
}

// the main stream has joined every side-stream merge issued so far: their result counters become
// ordinary pending counters (covered by the next read-back), their inputs are let go
static void side_outputs_joined(mzgpu_ctx* ctx) {
  std::vector<mzgpu_batch*> outs;
  outs.swap(ctx->side_outputs);
  for (auto* o : outs) {
    if (!o->st.known) o->st.seq = ++ctx->op_seq;
    mzgpu_batch *a = o->src1, *b = o->src2;
    o->src1 = o->src2 = nullptr;
    if (a) batch_release_internal(a);
    if (b) batch_release_internal(b);
    batch_release_internal(o);  // the list's reference
  }
}
// what a reader uses in place of `b`: the batch itself, or -- while its merge is still in flight on the
// side stream -- the merge's inputs (recursively)
static void expand_readable(mzgpu_batch* b, std::vector<mzgpu_batch*>& out) {
  if (b->side_seq > b->ctx->joined_seq && b->src1 != nullptr && b->src2 != nullptr) {
    expand_readable(b->src1, out);
    expand_readable(b->src2, out);
  } else {
    out.push_back(b);
  }
}
static int32_t batch_resolve(mzgpu_batch* b) {
  if (b->st.known) return MZGPU_OK;
  if (b->side_seq > b->ctx->joined_seq) {
    // its counters are written by a merge on the side stream
    if (b->ctx->stream == b->ctx->main_stream)
      MZ_TRY(mz_join_side(b->ctx));
    else if (b->st.seq == ~0ull)
      b->st.seq = ++b->ctx->op_seq;  // asked from the side stream itself: ordered behind that merge
  }
  MZ_TRY(b->st.resolve());
  b->len_ub = b->st.v[0];
  return MZGPU_OK;
}
// exact length (waits for the device if the batch is still in flight)
static u64 blen(mzgpu_batch* b) {
  if (batch_resolve(b) != MZGPU_OK) return 0;
  return b->st.v[0];
}
static DLen batch_dlen(const mzgpu_batch* b) { return dlen_of(b->st, 0); }

// sorted + consolidated device rows of known length -> indexed immutable batch
static int32_t make_batch(mzgpu_ctx* ctx, uint32_t rb, DevMem&& rows, u64 len, mzgpu_desc desc,
                          mzgpu_batch** out) {
  std::unique_ptr<mzgpu_batch> b(new mzgpu_batch());
  b->ctx = ctx;
  b->rb = rb;
  b->rows_cap = rows.bytes / rb;
  b->rows = std::move(rows);
  b->len_ub = len;
  b->desc = desc;
  u64 n_keys = 0, max_run = 0, slots = 0;
  MZ_TRY(mz_count_keys(ctx, rb, b->rows.p, len, &n_keys, &max_run));
  MZ_TRY(mz_build_index(ctx, rb, b->rows.p, len, n_keys, &b->table, &slots));
  b->st.set(ctx, len, slots - 1, n_keys, max_run);
  *out = b.release();
  return MZGPU_OK;
}
static int32_t batch_from_fused(mzgpu_ctx* ctx, uint32_t rb, FusedOut&& fo, u64 len_ub, mzgpu_desc desc,
                                mzgpu_batch** out) {
  mzgpu_batch* b = new mzgpu_batch();
  b->ctx = ctx;
  b->rb = rb;
  b->rows = std::move(fo.rows);
  b->rows_cap = fo.rows_cap;
  b->table = std::move(fo.table);
  b->st = std::move(fo.st);
  b->len_ub = len_ub;
  b->desc = desc;
  *out = b;
  return MZGPU_OK;
}
// Release the slack of a batch built with a loose capacity (its length is known now).
static int32_t batch_shrink(mzgpu_batch* b) {
  if (!b->st.known) return MZGPU_OK;
  MZ_TRY(batch_ready(b));
  mzgpu_ctx* ctx = b->ctx;
  const u64 len = b->st.v[0];
  const u64 slots_now = b->st.v[1] + 1;
  const bool realloc_rows = b->rows_cap > len + len / 2 + 4096;
  const bool realloc_table = b->table.p != nullptr && b->table.bytes > 2 * slots_now * sizeof(HashSlot) + 65536;
  // the old allocations are freed in stream order, i.e. AHEAD of jobs that were prepared but not
  // launched yet; such a job may read this batch (a deferred merge's input): launch them first
  if ((realloc_rows || realloc_table) && ctx->deferred_unlaunched > 0) MZ_TRY(mz_flush_deferred(ctx));
  if (realloc_rows) {
    DevMem m;
    MZ_TRY(m.alloc(ctx, std::max<u64>(len, 1) * b->rb, true));
    MZ_TRY(copy_in(ctx, m.p, b->rows.p, len * b->rb, MZGPU_MEM_DEVICE));
    b->rows = std::move(m);
    b->rows_cap = std::max<u64>(len, 1);
  }
  const u64 slots = b->st.v[1] + 1;
  if (b->table.p != nullptr && b->table.bytes > 2 * slots * sizeof(HashSlot) + 65536) {
    DevMem t;
    MZ_TRY(t.alloc(ctx, slots * sizeof(HashSlot), true));
    MZ_TRY(copy_in(ctx, t.p, b->table.p, slots * sizeof(HashSlot), MZGPU_MEM_DEVICE));
    b->table = std::move(t);
  }
  return MZGPU_OK;
}
// unsorted device rows -> batch
static int32_t build_batch_from_unsorted(mzgpu_ctx* ctx, uint32_t rb, const void* d_in, DLen n, u64 n_ub,
                                         mzgpu_desc desc, mzgpu_batch** out) {
  if (mz_use_fused(n.p == nullptr, n_ub)) {
    FusedJob job;
    job.rb = rb;
    job.a = d_in;
    job.na = n;
    job.cap = n_ub;
    job.want_index = true;
    FusedOut fo;
    MZ_TRY(mz_fused_consolidate(ctx, job, &fo));
    return batch_from_fused(ctx, rb, std::move(fo), n_ub, desc, out);
  }
  DevMem cons;
  u64 cap = 0;
  Lazy4 len;
  MZ_TRY(consolidate_dev(ctx, rb, d_in, n, n_ub, &cons, &cap, &len));
  MZ_TRY(len.resolve());
  return make_batch(ctx, rb, std::move(cons), len.v[0], desc, out);
}
static int32_t make_empty_batch(mzgpu_ctx* ctx, uint32_t rb, mzgpu_desc desc, mzgpu_batch** out) {
  mzgpu_batch* b = new mzgpu_batch();
  b->ctx = ctx;
  b->rb = rb;
  b->desc = desc;
  b->st.set(ctx, 0, 1, 0, 0);
  *out = b;
  MZ_TRY(b->rows.alloc(ctx, 16));
  b->rows_cap = 0;
  MZ_TRY(b->table.alloc(ctx, 2 * sizeof(HashSlot)));
  MZ_CUDA(ctx, cudaMemsetAsync(b->table.p, 0, 2 * sizeof(HashSlot), ctx->stream));
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_batch_build(mzgpu_ctx* ctx, uint32_t row_bytes, const void* rows, uint64_t n,
                                     int32_t mem, mzgpu_desc desc, mzgpu_batch** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || (rows == nullptr && n) || !arrangement_row_bytes(row_bytes)) return MZGPU_E_INVALID;
  if (n == 0) return make_empty_batch(ctx, row_bytes, desc, out);
  DevMem in;
  const void* d_in = rows;
  if (mem == MZGPU_MEM_HOST && n) {
    MZ_TRY(in.alloc(ctx, n * row_bytes));
    MZ_TRY(copy_in(ctx, in.p, rows, n * row_bytes, mem));
    d_in = in.p;
  }
  ctx->stats.rows_in += n;
  return build_batch_from_unsorted(ctx, row_bytes, d_in, dlen_imm(n), n, desc, out);
}
extern "C" uint64_t mzgpu_batch_len(const mzgpu_batch* b) { return b ? blen(const_cast<mzgpu_batch*>(b)) : 0; }
extern "C" uint64_t mzgpu_batch_keys(const mzgpu_batch* b) {
  if (b == nullptr || batch_resolve(const_cast<mzgpu_batch*>(b)) != MZGPU_OK) return 0;
  return b->st.v[2];
}
extern "C" mzgpu_desc mzgpu_batch_desc(const mzgpu_batch* b) {
  mzgpu_desc d = {0, 0, 0};
  return b ? b->desc : d;
}
extern "C" void mzgpu_batch_retain(mzgpu_batch* b) {
  if (b) b->refs++;
}
static void batch_release_internal(mzgpu_batch* b) {
  if (b && --b->refs == 0) {
    batch_ready(b);  // its memory is freed in stream order on the current stream
    delete b;
  }
}
extern "C" void mzgpu_batch_release(mzgpu_batch* b) { batch_release_internal(b); }
extern "C" int32_t mzgpu_batch_export(mzgpu_batch* b, void* rows, uint64_t cap, int32_t mem,
                                      uint64_t* n_out) {
  if (b == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  MZ_TRY(batch_ready(b));
  MZ_TRY(batch_resolve(b));
  const u64 len = b->st.v[0];
  if (n_out) *n_out = len;
  if (cap < len) return MZGPU_E_CAPACITY;
  MZ_TRY(copy_out(b->ctx, rows, b->rows.p, len * b->rb, mem));
  return MZGPU_OK;
}
// ---- a8: batched cursor calls
extern "C" int32_t mzgpu_batch_seek_keys(mzgpu_batch* b, const uint64_t* keys, uint64_t n, int32_t mem,
                                         mzgpu_key_run* runs) {
  if (b == nullptr || (n && (keys == nullptr || runs == nullptr))) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = b->ctx;
  MZ_CHECK_CTX(ctx);
  if (n == 0) return MZGPU_OK;
  MZ_TRY(batch_ready(b));
  DevMem dk, dr;
  const u64* d_keys = keys;
  u64* d_runs = (u64*)runs;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(dk.alloc(ctx, n * 8));
    MZ_TRY(dr.alloc(ctx, n * sizeof(mzgpu_key_run)));
    MZ_TRY(copy_in(ctx, dk.p, keys, n * 8, mem));
    d_keys = dk.as<u64>();
    d_runs = dr.as<u64>();
  }
  MZ_TRY(mz_seek_keys(ctx, (int)b->rb, b->rows.p, batch_dlen(b), d_keys, n, d_runs));
  if (mem == MZGPU_MEM_HOST) MZ_TRY(copy_out(ctx, runs, d_runs, n * sizeof(mzgpu_key_run), mem));
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_batch_key_page(mzgpu_batch* b, uint64_t first_ordinal, uint64_t max_keys, int32_t mem,
                                        mzgpu_key_run* runs, uint64_t* n_out) {
  if (b == nullptr || (max_keys && runs == nullptr)) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = b->ctx;
  MZ_CHECK_CTX(ctx);
  MZ_TRY(batch_ready(b));
  MZ_TRY(batch_resolve(b));
  const u64 n_keys = b->st.v[2];
  u64 avail = first_ordinal < n_keys ? n_keys - first_ordinal : 0;
  if (avail > max_keys) avail = max_keys;
  if (n_out) *n_out = avail;
  if (avail == 0) return MZGPU_OK;
  DevMem dr;
  u64* d_runs = (u64*)runs;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(dr.alloc(ctx, avail * sizeof(mzgpu_key_run)));
    d_runs = dr.as<u64>();
  }
  MZ_TRY(mz_key_page(ctx, (int)b->rb, b->rows.p, b->st.v[0], first_ordinal, avail, d_runs));
  if (mem == MZGPU_MEM_HOST) MZ_TRY(copy_out(ctx, runs, d_runs, avail * sizeof(mzgpu_key_run), mem));
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_batch_rows(mzgpu_batch* b, uint64_t first, uint64_t len, void* rows, int32_t mem) {
  if (b == nullptr || (len && rows == nullptr)) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  if (len == 0) return MZGPU_OK;
  MZ_TRY(batch_ready(b));
  MZ_TRY(batch_resolve(b));
  if (first > b->st.v[0] || len > b->st.v[0] - first) {
    MZ_SET_ERR(b->ctx, "batch_rows: [%llu, +%llu) is outside the batch's %llu rows", (unsigned long long)first,
               (unsigned long long)len, (unsigned long long)b->st.v[0]);
    return MZGPU_E_INVALID;
  }
  return copy_out(b->ctx, rows, (const char*)b->rows.p + first * b->rb, len * b->rb, mem);
}
extern "C" int32_t mzgpu_batch_index_export(mzgpu_batch* b, void* slots, uint64_t cap_slots, int32_t mem,
                                            uint64_t* n_slots, uint64_t* n_keys, uint64_t* longest_run) {
  if (b == nullptr || (cap_slots && slots == nullptr)) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  MZ_TRY(batch_ready(b));
  MZ_TRY(batch_resolve(b));
  const u64 ns = b->st.v[1] + 1;
  if (n_slots) *n_slots = ns;
  if (n_keys) *n_keys = b->st.v[2];
  if (longest_run) *longest_run = b->st.v[3];
  if (cap_slots < ns) return MZGPU_E_CAPACITY;
  return copy_out(b->ctx, slots, b->table.p, ns * sizeof(HashSlot), mem);
}

// ---- a5: Builder::{push, done}
struct mzgpu_builder {
  mzgpu_ctx* ctx;
  uint32_t rb;
  mzgpu_buf rows;
};
extern "C" int32_t mzgpu_builder_new(mzgpu_ctx* ctx, uint32_t row_bytes, uint64_t capacity_rows,
                                     mzgpu_builder** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || !arrangement_row_bytes(row_bytes)) return MZGPU_E_INVALID;
  std::unique_ptr<mzgpu_builder> b(new mzgpu_builder());
  b->ctx = ctx;
  b->rb = row_bytes;
  b->rows.ctx = ctx;
  b->rows.rb = row_bytes;
  buf_set_len(&b->rows, 0);
  if (capacity_rows) MZ_TRY(buf_reserve(&b->rows, capacity_rows, false));
  *out = b.release();
  return MZGPU_OK;
}
extern "C" void mzgpu_builder_free(mzgpu_builder* b) { delete b; }
extern "C" int32_t mzgpu_builder_push(mzgpu_builder* b, const void* rows, uint64_t n, int32_t mem) {
  if (b == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  if (n == 0) return MZGPU_OK;
  if (mem == MZGPU_MEM_DEVICE) return buf_append_dev(&b->rows, rows, dlen_imm(n), n);
  MZ_TRY(buf_resolve(&b->rows));
  MZ_TRY(buf_reserve(&b->rows, b->rows.ub + n, true));
  MZ_TRY(copy_in(b->ctx, (char*)b->rows.mem.p + b->rows.ub * b->rb, rows, n * b->rb, mem));
  buf_set_len(&b->rows, b->rows.ub + n);
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_builder_push_buf(mzgpu_builder* b, mzgpu_buf* rows) {
  if (b == nullptr || rows == nullptr || rows->rb != b->rb) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  return buf_append_dev(&b->rows, rows->mem.p, buf_dlen(rows), rows->ub);
}
extern "C" int32_t mzgpu_builder_done(mzgpu_builder* b, mzgpu_desc desc, mzgpu_batch** out) {
  if (b == nullptr || out == nullptr) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = b->ctx;
  MZ_CHECK_CTX(ctx);
  int32_t st;
  if (b->rows.ub == 0) {
    st = make_empty_batch(ctx, b->rb, desc, out);
  } else {
    ctx->stats.rows_in += b->rows.ub;
    st = build_batch_from_unsorted(ctx, b->rb, b->rows.mem.p, buf_dlen(&b->rows), b->rows.ub, desc, out);
  }
  buf_set_len(&b->rows, 0);  // (the storage is kept for the next batch; the build read it in stream order)
  return st;
}

// Batch::Merger in one step: union, advance_by(since), consolidate, index.
static int32_t merge_batches(mzgpu_batch* b1, mzgpu_batch* b2, u64 since, mzgpu_batch** out) {
  mzgpu_ctx* ctx = b1->ctx;
  // an input that is itself the output of a deferred merge must be launched first (jobs of one
  // multi-job launch run side by side)
  MZ_TRY(batch_ready(b1));
  MZ_TRY(batch_ready(b2));
  mzgpu_desc d = {b1->desc.lower, b2->desc.upper, since};
  // advance_by of an empty antichain leaves every time alone (SURVEY A4); the kernels compute
  // max(time, since), for which 0 is the no-op
  const u64 adv = since == MZGPU_FRONTIER_EMPTY ? 0 : since;
  // R32 arrangements: the merge-path kernels (mergepath.cu) -- three ordinary launches, any size, no
  // host wait, no cooperative launch
  if (b1->rb == 32 && (b1->len_ub + b2->len_ub + 1023) / 1024 <= MZ_LB_TILES) {
    const u64 cap = b1->len_ub + b2->len_ub;
    FusedOut fo;
    MZ_TRY(mz_merge_r32_async(ctx, b1->rows.p, batch_dlen(b1), b2->rows.p, batch_dlen(b2), cap, adv, &fo));
    return batch_from_fused(ctx, 32, std::move(fo), cap, d, out);
  }
  if (!mz_use_fused(false, b1->len_ub + b2->len_ub)) {
    MZ_TRY(batch_resolve(b1));
    MZ_TRY(batch_resolve(b2));
  }
  if (mz_use_fused(b1->st.known && b2->st.known, b1->len_ub + b2->len_ub)) {
    FusedJob job;
    job.rb = b1->rb;
    job.a = b1->rows.p;
    job.na = batch_dlen(b1);
    job.b = b2->rows.p;
    job.nb = batch_dlen(b2);
    job.cap = b1->len_ub + b2->len_ub;
    job.since = adv;
    job.want_index = true;
    job.merge = true;
    FusedOut fo;
    if (ctx->stream == ctx->main_stream) {
      // The merges that the inserts of one timestamp trigger (one per arrangement, all alike)
      // are independent: they are prepared here and launched together, by the first reader of
      // any of their outputs (batch_ready) or the next counter read-back.
      MZ_TRY(mz_fused_defer(ctx, job, &fo));
      b1->refs++;
      b2->refs++;
      ctx->deferred_inputs.push_back(b1);
      ctx->deferred_inputs.push_back(b2);
      const u64 seq = ++ctx->defer_seq;
      MZ_TRY(batch_from_fused(ctx, b1->rb, std::move(fo), job.cap, d, out));
      (*out)->deferred_seq = seq;
      return MZGPU_OK;
    }
    MZ_TRY(mz_fused_consolidate(ctx, job, &fo));
    return batch_from_fused(ctx, b1->rb, std::move(fo), job.cap, d, out);
  }
  MZ_TRY(batch_resolve(b1));
  MZ_TRY(batch_resolve(b2));
  DevMem merged;
  u64 n_out = 0;
  MZ_TRY(mz_merge_consolidate(ctx, b1->rb, b1->rows.p, b1->st.v[0], b2->rows.p, b2->st.v[0], adv, &merged,
                              &n_out));
  return make_batch(ctx, b1->rb, std::move(merged), n_out, d, out);
}
extern "C" int32_t mzgpu_batch_merge(mzgpu_batch* b1, mzgpu_batch* b2, uint64_t since,
                                     mzgpu_batch** out) {
  if (b1 == nullptr || b2 == nullptr || out == nullptr || b1->rb != b2->rb) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b1->ctx);
  if (b1->desc.upper != b2->desc.lower) {
    MZ_SET_ERR(b1->ctx, "batch_merge: b1.upper %llu != b2.lower %llu", (unsigned long long)b1->desc.upper,
               (unsigned long long)b2->desc.lower);
    return MZGPU_E_FRONTIER;
  }
  MZ_TRY(batch_ready(b1));
  MZ_TRY(batch_ready(b2));
  return merge_batches(b1, b2, since, out);
}

// ================================================================== batcher
// The reference's MergeBatcher sorts every pushed container at once and keeps
// geometric chains of sorted chunks, merging them at seal time.  On the GPU the
// cheaper schedule is to stash pushed containers as they are and do all the
// work at seal: ONE sort + consolidate of everything buffered, split by the
// seal frontier (ship: time < upper; keep: the rest) and index of the shipped
// rows — a single fused kernel for update batches.  The sealed batches and the
// batcher frontier are identical to the reference's; only the moment the
// sorting happens differs.  The stash is compacted when it grows large.
struct Seg {
  DevMem rows;
  Lazy4 len;  // word `word` = rows; for the keep segment of a seal: [0] rows, [1] min kept time
  int word = 0;
  u64 ub = 0;
  bool is_keep = false;
};
struct mzgpu_batcher {
  mzgpu_ctx* ctx;
  uint32_t rb;
  std::vector<Seg> segs;
  u64 lower = 0;
  bool frontier_known = true;  // else: derived from the keep segment segs[0]
  u64 frontier = MZGPU_FRONTIER_EMPTY;
};
#define MZ_STASH_COMPACT_ROWS (64ull << 20)

static u64 batcher_ub(const mzgpu_batcher* b) {
  u64 n = 0;
  for (auto& s : b->segs) n += s.ub;
  return n;
}
static int32_t batcher_resolve_frontier(mzgpu_batcher* b) {
  if (b->frontier_known) return MZGPU_OK;
  Seg& k = b->segs[0];
  if (!k.len.known) {
    MZ_TRY(k.len.resolve());
    k.ub = k.len.v[0];
  }
  b->frontier = k.len.v[0] ? k.len.v[1] : MZGPU_FRONTIER_EMPTY;
  b->frontier_known = true;
  return MZGPU_OK;
}
// all segments into one device array (device-side offsets where lengths are pending)
static int32_t batcher_concat(mzgpu_batcher* b, DevMem* out, Lazy4* out_len, int* out_word, u64* out_ub) {
  mzgpu_ctx* ctx = b->ctx;
  const u64 total = batcher_ub(b);
  MZ_TRY(out->alloc(ctx, std::max<u64>(total, 1) * b->rb));
  mzgpu_buf tmp;  // borrow the append logic of a buffer
  tmp.ctx = ctx;
  tmp.rb = b->rb;
  tmp.mem = std::move(*out);
  tmp.cap = std::max<u64>(total, 1);
  tmp.len.set(ctx, 0);
  for (auto& s : b->segs) MZ_TRY(buf_append_dev(&tmp, s.rows.p, dlen_of(s.len, s.word), s.ub));
  *out = std::move(tmp.mem);
  *out_len = std::move(tmp.len);
  *out_word = tmp.word;
  *out_ub = tmp.ub;
  return MZGPU_OK;
}
static int32_t batcher_push_seg(mzgpu_batcher* b, Seg&& s) {
  if (s.ub == 0) return MZGPU_OK;
  b->segs.push_back(std::move(s));
  if (batcher_ub(b) > MZ_STASH_COMPACT_ROWS && b->segs.size() > 1) {
    // compact the stash: consolidate everything buffered into one segment
    MZ_TRY(batcher_resolve_frontier(b));
    DevMem all, cons;
    Lazy4 len, clen;
    int word = 0;
    u64 ub = 0, cap = 0;
    MZ_TRY(batcher_concat(b, &all, &len, &word, &ub));
    MZ_TRY(consolidate_dev(b->ctx, b->rb, all.p, dlen_of(len, word), ub, &cons, &cap, &clen));
    MZ_TRY(clen.resolve());
    b->segs.clear();
    Seg c;
    c.rows = std::move(cons);
    c.ub = clen.v[0];
    c.len.set(b->ctx, clen.v[0]);
    b->segs.push_back(std::move(c));
  }
  return MZGPU_OK;
}
// push device rows the batcher may keep a pointer to only by copying
static int32_t batcher_push_dev(mzgpu_batcher* b, const void* d_rows, DLen n, u64 n_ub) {
  if (n_ub == 0) return MZGPU_OK;
  Seg s;
  MZ_TRY(s.rows.alloc(b->ctx, n_ub * b->rb));
  if (n.p == nullptr) {
    MZ_TRY(copy_in(b->ctx, s.rows.p, d_rows, n.imm * b->rb, MZGPU_MEM_DEVICE));
    s.len.set(b->ctx, n.imm);
    s.ub = n.imm;
  } else {
    MZ_TRY(s.len.make_pending(b->ctx));
    MZ_TRY(append_dev(b->ctx, d_rows, n, n_ub, b->rb, s.rows.p, dlen_imm(0), n_ub, s.len.dptr()));
    s.len.mark_written();
    s.ub = n_ub;
  }
  return batcher_push_seg(b, std::move(s));
}
// A seal in three steps, so that the fused launches of several batchers sealed at the same
// frontier can share one cooperative launch (seal_many): plan (what to run) -> run -> finish.
struct SealPlan {
  mzgpu_batcher* b = nullptr;
  u64 upper = 0;
  mzgpu_desc d = {0, 0, 0};
  u64 total = 0;
  bool exact = true;
  bool fused = false;  // one fused job (`job`) does the whole seal
  DevMem all;          // concatenated stash (kept alive until the launch is enqueued)
  Lazy4 alen;
  FusedJob job;
  FusedOut fo;
};

static int32_t seal_plan(mzgpu_batcher* b, u64 upper, SealPlan* p) {
  mzgpu_ctx* ctx = b->ctx;
  if (upper != MZGPU_FRONTIER_EMPTY && upper < b->lower) {
    MZ_SET_ERR(ctx, "batcher_seal: upper %llu precedes lower %llu", (unsigned long long)upper,
               (unsigned long long)b->lower);
    return MZGPU_E_FRONTIER;
  }
  // segments known to be empty cost nothing
  {
    std::vector<Seg> live;
    for (auto& s : b->segs) {
      // a count that has already reached the host (some read-back happened since) costs nothing
      if (s.len.try_resolve()) s.ub = s.len.v[s.word];
      if (!(s.len.known && s.len.v[s.word] == 0)) live.push_back(std::move(s));
    }
    b->segs = std::move(live);
  }
  p->b = b;
  p->upper = upper;
  p->d = mzgpu_desc{b->lower, upper, 0};
  bool exact = true;
  for (auto& s : b->segs) exact = exact && s.len.known;
  if (!exact && !mz_use_fused(false, batcher_ub(b))) {
    for (auto& s : b->segs) {
      MZ_TRY(s.len.resolve());
      s.ub = s.len.v[s.word];
    }
    exact = true;
  }
  p->exact = exact;
  p->total = batcher_ub(b);
  p->fused = p->total > 0 && mz_use_fused(exact, p->total);
  if (p->fused) {
    int aword = 0;
    u64 aub = 0;
    p->job.rb = b->rb;
    if (b->segs.size() == 1) {
      p->job.a = b->segs[0].rows.p;
      p->job.na = dlen_of(b->segs[0].len, b->segs[0].word);
    } else {
      MZ_TRY(batcher_concat(b, &p->all, &p->alen, &aword, &aub));
      p->job.a = p->all.p;
      p->job.na = dlen_of(p->alen, aword);
    }
    p->job.cap = p->total;
    p->job.upper = upper;
    p->job.want_index = true;
  }
  return MZGPU_OK;
}

// after the fused launch of the plan has been enqueued
static int32_t seal_finish_fused(SealPlan* p, mzgpu_batch** batch_out) {
  mzgpu_batcher* b = p->b;
  mzgpu_ctx* ctx = b->ctx;
  b->segs.clear();  // stream ordered: the kernel still reads them
  if (p->upper != MZGPU_FRONTIER_EMPTY) {
    Seg k;
    k.rows = std::move(p->fo.keep);
    k.len = std::move(p->fo.kst);
    k.word = 0;
    k.ub = p->total;
    k.is_keep = true;
    b->segs.push_back(std::move(k));
    b->frontier_known = false;
  } else {
    b->frontier = MZGPU_FRONTIER_EMPTY;
    b->frontier_known = true;
  }
  return batch_from_fused(ctx, b->rb, std::move(p->fo), p->total, p->d, batch_out);
}

// the seals a fused job cannot take: nothing buffered, or the bulk multi-kernel path
static int32_t seal_run_unfused(SealPlan* p, mzgpu_batch** batch_out) {
  mzgpu_batcher* b = p->b;
  mzgpu_ctx* ctx = b->ctx;
  const u64 upper = p->upper;
  const mzgpu_desc d = p->d;
  if (p->total == 0) {
    b->segs.clear();
    b->frontier = MZGPU_FRONTIER_EMPTY;
    b->frontier_known = true;
    return make_empty_batch(ctx, b->rb, d, batch_out);
  }
  // bulk path: exact sizes, multi-kernel sort / extract
  DevMem all, cons;
  Lazy4 alen, clen;
  int aword = 0;
  u64 aub = 0, cap = 0;
  const void* src = nullptr;
  DLen sn;
  if (b->segs.size() == 1) {
    src = b->segs[0].rows.p;
    sn = dlen_of(b->segs[0].len, b->segs[0].word);
    aub = b->segs[0].ub;
  } else {
    MZ_TRY(batcher_concat(b, &all, &alen, &aword, &aub));
    src = all.p;
    sn = dlen_of(alen, aword);
  }
  ctx->last_minmax_valid = false;
  MZ_TRY(consolidate_dev(ctx, b->rb, src, sn, aub, &cons, &cap, &clen));
  MZ_TRY(clen.resolve());
  b->segs.clear();
  all.release();
  const u64 n_cons = clen.v[0];
  b->frontier = MZGPU_FRONTIER_EMPTY;
  b->frontier_known = true;
  // the bulk sort has seen the range of the time word: if every buffered time precedes
  // `upper` everything ships and the extract pass (two more copies of the rows) is skipped
  const int tw = b->rb == 32 ? 2 : (b->rb == 72 ? RowT<72>::TW : (b->rb == 40 ? RowT<40>::TW : 1));
  const bool all_ship = ctx->last_minmax_valid && ctx->last_minmax[2 * tw + 1] < upper;
  if (upper == MZGPU_FRONTIER_EMPTY || n_cons == 0 || all_ship) {
    MZ_TRY(make_batch(ctx, b->rb, std::move(cons), n_cons, d, batch_out));
  } else {
    DevMem ship, keep;
    u64 n_ship = 0, n_keep = 0, min_keep = MZGPU_FRONTIER_EMPTY;
    MZ_TRY(mz_extract(ctx, b->rb, cons.p, n_cons, upper, &ship, &n_ship, &keep, &n_keep, &min_keep));
    cons.release();
    if (n_keep) {
      Seg k;
      k.rows = std::move(keep);
      k.len.set(ctx, n_keep);
      k.ub = n_keep;
      b->segs.push_back(std::move(k));
      b->frontier = min_keep;
    }
    MZ_TRY(make_batch(ctx, b->rb, std::move(ship), n_ship, d, batch_out));
  }
  return MZGPU_OK;
}

static int32_t batcher_seal(mzgpu_batcher* b, u64 upper, mzgpu_batch** batch_out, u64* new_lower) {
  SealPlan p;
  MZ_TRY(seal_plan(b, upper, &p));
  if (p.fused) {
    MZ_TRY(mz_fused_consolidate(b->ctx, p.job, &p.fo));
    MZ_TRY(seal_finish_fused(&p, batch_out));
  } else {
    MZ_TRY(seal_run_unfused(&p, batch_out));
  }
  b->lower = upper;
  if (new_lower) {
    MZ_TRY(batcher_resolve_frontier(b));
    *new_lower = b->frontier;
  }
  return MZGPU_OK;
}

// Seal k batchers at the same frontier; the fused jobs of one row width share ONE cooperative
// launch (groups of MZ_FUSED_MANY_MAX).  Same results as k batcher_seal calls in this order.
static int32_t batcher_seal_many(int k, mzgpu_batcher* const* bs, u64 upper, mzgpu_batch** batches_out) {
  if (k <= 0) return MZGPU_OK;
  std::vector<SealPlan> plans((size_t)k);
  for (int i = 0; i < k; ++i) {
    batches_out[i] = nullptr;
    MZ_TRY(seal_plan(bs[i], upper, &plans[(size_t)i]));
  }
  std::vector<char> done((size_t)k, 0);
  for (int i = 0; i < k; ++i) {
    if (done[(size_t)i] || !plans[(size_t)i].fused) continue;
    // this plan and the later fused plans of the same row width
    int idx[MZ_FUSED_MANY_MAX];
    int g = 0;
    for (int j = i; j < k && g < MZ_FUSED_MANY_MAX; ++j)
      if (!done[(size_t)j] && plans[(size_t)j].fused && plans[(size_t)j].job.rb == plans[(size_t)i].job.rb) idx[g++] = j;
    FusedJob jobs[MZ_FUSED_MANY_MAX];
    FusedOut outs[MZ_FUSED_MANY_MAX];
    for (int t = 0; t < g; ++t) jobs[t] = plans[(size_t)idx[t]].job;
    MZ_TRY(mz_fused_consolidate_many(bs[i]->ctx, g, jobs, outs));
    for (int t = 0; t < g; ++t) {
      plans[(size_t)idx[t]].fo = std::move(outs[t]);
      done[(size_t)idx[t]] = 1;
    }
  }
  for (int i = 0; i < k; ++i) {
    SealPlan& p = plans[(size_t)i];
    if (p.fused)
      MZ_TRY(seal_finish_fused(&p, &batches_out[i]));
    else
      MZ_TRY(seal_run_unfused(&p, &batches_out[i]));
    bs[i]->lower = upper;
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_batcher_new(mzgpu_ctx* ctx, uint32_t row_bytes, mzgpu_batcher** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || !arrangement_row_bytes(row_bytes)) return MZGPU_E_INVALID;
  mzgpu_batcher* b = new mzgpu_batcher();
  b->ctx = ctx;
  b->rb = row_bytes;
  *out = b;
  return MZGPU_OK;
}
extern "C" void mzgpu_batcher_free(mzgpu_batcher* b) { delete b; }
extern "C" int32_t mzgpu_batcher_push(mzgpu_batcher* b, const void* rows, uint64_t n, int32_t mem) {
  if (b == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  if (n == 0) return MZGPU_OK;
  b->ctx->stats.rows_in += n;
  if (mem == MZGPU_MEM_HOST) {
    Seg s;
    MZ_TRY(s.rows.alloc(b->ctx, n * b->rb));
    MZ_TRY(copy_in(b->ctx, s.rows.p, rows, n * b->rb, mem));
    s.len.set(b->ctx, n);
    s.ub = n;
    return batcher_push_seg(b, std::move(s));
  }
  return batcher_push_dev(b, rows, dlen_imm(n), n);
}
extern "C" int32_t mzgpu_batcher_push_buf(mzgpu_batcher* b, mzgpu_buf* rows) {
  if (b == nullptr || rows == nullptr || rows->rb != b->rb) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  b->ctx->stats.rows_in += rows->ub;
  return batcher_push_dev(b, rows->mem.p, buf_dlen(rows), rows->ub);
}
extern "C" int32_t mzgpu_batcher_seal(mzgpu_batcher* b, uint64_t upper, mzgpu_batch** batch_out,
                                      uint64_t* new_lower) {
  if (b == nullptr || batch_out == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(b->ctx);
  return batcher_seal(b, upper, batch_out, new_lower);
}
extern "C" int32_t mzgpu_batcher_seal_many(uint32_t k, mzgpu_batcher* const* batchers, uint64_t upper,
                                           mzgpu_batch** batches_out) {
  if (k == 0) return MZGPU_OK;
  if (batchers == nullptr || batches_out == nullptr) return MZGPU_E_INVALID;
  for (uint32_t i = 0; i < k; ++i) {
    if (batchers[i] == nullptr || batchers[i]->ctx != batchers[0]->ctx) return MZGPU_E_INVALID;
    for (uint32_t j = 0; j < i; ++j)
      if (batchers[j] == batchers[i]) return MZGPU_E_INVALID;
  }
  MZ_CHECK_CTX(batchers[0]->ctx);
  return batcher_seal_many((int)k, batchers, upper, batches_out);
}
extern "C" uint64_t mzgpu_batcher_frontier(const mzgpu_batcher* b) {
  if (b == nullptr) return MZGPU_FRONTIER_EMPTY;
  if (batcher_resolve_frontier(const_cast<mzgpu_batcher*>(b)) != MZGPU_OK) return MZGPU_FRONTIER_EMPTY;
  return b->frontier;
}
// Updates currently buffered (as pushed: the stash is consolidated at seal).
extern "C" uint64_t mzgpu_batcher_len(const mzgpu_batcher* cb) {
  mzgpu_batcher* b = const_cast<mzgpu_batcher*>(cb);
  u64 n = 0;
  if (b)
    for (auto& s : b->segs) {
      if (!s.len.known) {
        if (s.len.resolve() != MZGPU_OK) return 0;
        s.ub = s.len.v[s.word];
      }
      n += s.len.v[s.word];
    }
  return n;
}

// ==================================================================== spine
// Host-side restatement of spine_fueled::Spine's scheduling (in-tree fork
// src/persist-client/src/internal/trace.rs:1565-2262; SURVEY.md A5) over
// device batches.  Fuel is bookkeeping on the host; a merge runs as one kernel
// sequence when the schedule completes it.  Batches whose length is still in
// flight on the device wait in `pending` (they are visible to readers, as any
// inserted batch is) and are admitted to the layers — which need exact lengths —
// when physical compaction allows it.
struct mzgpu_spine {
  struct Layer {
    std::vector<mzgpu_batch*> batches;  // at most 2 (owned references)
    bool has_merge = false;
    u64 merge_since = 0;
    u64 remaining = 0;
    // The work of a merge is the exact length of its inputs.  An input that was itself
    // just produced by a merge still has its length on the device; rather than wait for
    // it, the fuel applied meanwhile is remembered and `remaining` is settled later
    // (remaining = max(0, work - fuel applied), exactly what repeated saturating
    // subtraction gives), unless the decision "does this fuel complete the merge?"
    // really depends on the unknown length.
    bool lazy_work = false;
    u64 fuel_debt = 0;
  };
  // settle a lazily accounted merge; returns false if a length is still on the device
  static bool settle(Layer& m, bool force) {
    if (!m.lazy_work) return true;
    for (auto* b : m.batches)
      if (!b->st.known) {
        if (b->st.try_resolve())
          b->len_ub = b->st.v[0];
        else if (force)
          blen(b);
        else
          return false;
      }
    u64 work = 0;
    for (auto* b : m.batches) work += b->st.v[0];
    m.remaining = work - std::min(work, m.fuel_debt);
    m.lazy_work = false;
    m.fuel_debt = 0;
    return true;
  }
  mzgpu_ctx* ctx;
  uint32_t rb;
  u64 effort = 1;
  u64 since = 0;
  u64 physical = 0;
  u64 upper = 0;
  std::vector<Layer> merging;
  std::vector<mzgpu_batch*> pending;  // not yet admitted (upper > physical compaction)
  std::vector<mzgpu_batch*> view;     // scratch for batches_through
  int32_t err = MZGPU_OK;             // first failure inside a scheduling step

  // usize::next_power_of_two().trailing_zeros() (trace.rs:1714); next_power_of_two overflows
  // beyond 2^63 in the reference (a debug panic / release 0): capped at level 63 here
  static u64 level_of(u64 n) {
    if (n <= 1) return 0;
    const u64 l = 64 - (u64)__builtin_clzll(n - 1);
    return l > 63 ? 63 : l;
  }
  u64 layer_len(const Layer& m) const {
    u64 n = 0;
    for (auto* b : m.batches) n += blen(b);
    return n;
  }
  bool reduced() const {
    int non_empty = 0;
    for (auto& m : merging) {
      if (m.batches.size() == 2) return false;
      if (layer_len(m) > 0) ++non_empty;
      if (non_empty > 1) return false;
    }
    return true;
  }
  void begin_merge(Layer& m, bool with_frontier) {
    u64 s = 0;
    for (auto* b : m.batches) s = std::max(s, b->desc.since);
    if (with_frontier) s = std::max(s, since);
    m.has_merge = true;
    m.merge_since = s;
    m.lazy_work = true;
    m.fuel_debt = 0;
    m.remaining = 0;
    settle(m, false);
  }
  void insert_at(mzgpu_batch* b, size_t index) {
    while (merging.size() <= index) merging.push_back(Layer());
    Layer& m = merging[index];
    if (m.has_merge || m.batches.size() >= 2) {
      MZ_SET_ERR(ctx, "spine: attempted to insert batch into a full / merging layer %zu", index);
      err = MZGPU_E_INVALID;
      mzgpu_batch_release(b);
      return;
    }
    m.batches.push_back(b);
    if (m.batches.size() == 2) begin_merge(m, true);
  }
  // MergeState::complete: returns an owned batch or nullptr
  mzgpu_batch* complete_at(size_t index) {
    Layer m = std::move(merging[index]);
    merging[index] = Layer();
    if (m.batches.empty()) return nullptr;
    if (m.batches.size() == 1) return m.batches[0];
    if (!m.has_merge) begin_merge(m, false);
    mzgpu_batch *b1 = m.batches[0], *b2 = m.batches[1];
    mzgpu_batch* out = nullptr;
    int32_t st;
    if (b1->st.known && b2->st.known && b1->st.v[0] == 0 && b2->st.v[0] == 0) {
      mzgpu_desc d = {b1->desc.lower, b2->desc.upper, m.merge_since};
      st = make_empty_batch(ctx, rb, d, &out);
    } else if (ctx->stream == ctx->main_stream && !ctx->profile && rb == 32) {
      // Spine maintenance runs on the side stream, concurrently with the operators on the main
      // stream (the merge-path kernels are ordinary launches: they share the machine with the probes
      // and the reduce of the timestamp that triggered them).  The side stream first catches up with
      // the main stream (the inputs are ordered before it).  The inputs stay alive, and VISIBLE TO
      // READERS in place of the output, until the main stream joins the merge (expand_readable).
      cudaEventRecord(ctx->ev_fork, ctx->main_stream);
      cudaStreamWaitEvent(ctx->side_stream, ctx->ev_fork, 0);
      mz_mid_forked(ctx);
      ctx->stream = ctx->side_stream;
      st = merge_batches(b1, b2, m.merge_since, &out);
      cudaEventRecord(ctx->ev_side, ctx->side_stream);
      ctx->stream = ctx->main_stream;
      ctx->side_seq++;
      if (out != nullptr) {
        out->side_seq = ctx->side_seq;
        if (!out->st.known) out->st.seq = ~0ull;  // not covered by a read-back before the join
        out->src1 = b1;  // (the references this function holds move to the output)
        out->src2 = b2;
        b1 = b2 = nullptr;
        out->refs++;
        ctx->side_outputs.push_back(out);
      }
    } else {
      st = merge_batches(b1, b2, m.merge_since, &out);
    }
    if (st != MZGPU_OK && err == MZGPU_OK) err = st;
    if (b1) mzgpu_batch_release(b1);
    if (b2) mzgpu_batch_release(b2);
    return out;
  }
  void apply_fuel(long long fuel_in) {
    for (size_t index = 0; index < merging.size(); ++index) {
      Layer& m = merging[index];
      if (m.has_merge) {
        u64 f = fuel_in < 0 ? 0 : (u64)fuel_in;
        if (m.lazy_work && !settle(m, false)) {
          // bounds on the work: unknown lengths lie in [0, len_ub]
          u64 lo = 0, hi = 0;
          for (auto* b : m.batches) {
            lo += b->st.known ? b->st.v[0] : 0;
            hi += b->st.known ? b->st.v[0] : b->len_ub;
          }
          const u64 total = m.fuel_debt + f;
          if (total >= hi) {
            m.lazy_work = false;  // completes whatever the exact length is
            m.remaining = 0;
            f = 0;
          } else if (total < lo) {
            m.fuel_debt = total;  // cannot complete yet: settle later
            continue;
          } else {
            settle(m, true);  // the decision depends on the exact length
          }
        }
        m.remaining -= std::min(f, m.remaining);
      }
      if (m.has_merge && m.remaining == 0) {
        mzgpu_batch* done = complete_at(index);
        if (done) insert_at(done, index + 1);
      }
    }
  }
  void roll_up(size_t index) {
    while (merging.size() <= index) merging.push_back(Layer());
    bool any = false;
    for (size_t i = 0; i < index; ++i) any = any || !merging[i].batches.empty();
    if (!any) return;
    mzgpu_batch* merged = nullptr;
    for (size_t i = 0; i < index; ++i) {
      if (merged) {
        insert_at(merged, i);
        merged = nullptr;
      }
      merged = complete_at(i);
    }
    if (merged) insert_at(merged, index);
    if (merging[index].batches.size() == 2) {
      mzgpu_batch* m2 = complete_at(index);
      if (m2) insert_at(m2, index + 1);
    }
  }
  void tidy_layers() {
    if (merging.empty()) return;
    size_t length = merging.size();
    if (merging[length - 1].batches.size() != 1) return;
    u64 appropriate = level_of(layer_len(merging[length - 1]));
    while (appropriate < length - 1) {
      Layer& cur = merging[length - 2];
      if (cur.batches.empty()) {
        merging.erase(merging.begin() + (length - 2));
        length = merging.size();
      } else {
        if (cur.batches.size() != 2) {
          u64 smaller = 0;
          for (size_t i = 0; i < length - 2; ++i) smaller += (u64)merging[i].batches.size() << i;
          if (smaller <= ((u64)1 << length) / 8) {
            Layer state = std::move(merging[length - 2]);
            merging.erase(merging.begin() + (length - 2));
            for (auto* b : state.batches) insert_at(b, length - 2);
          }
        }
        break;
      }
    }
  }
  void introduce_batch(mzgpu_batch* b, size_t index) {
    long long fuel = (long long)((8ull << index) * effort);
    apply_fuel(fuel);
    roll_up(index);
    insert_at(b, index);
    tidy_layers();
  }
  void insert_entry(mzgpu_batch* b) {
    if (blen(b) == 0) {
      for (size_t pos = 0; pos < merging.size(); ++pos) {
        if (merging[pos].batches.empty()) continue;
        if (merging[pos].batches.size() == 1 && layer_len(merging[pos]) == 0) {
          insert_at(b, pos);
          mzgpu_batch* merged = complete_at(pos);
          if (merged) {
            merging[pos] = Layer();
            merging[pos].batches.push_back(merged);
          }
          return;
        }
        break;
      }
    }
    introduce_batch(b, level_of(blen(b)));
  }
  void consider_merges() {
    while (!pending.empty()) {
      mzgpu_batch* b = pending.front();
      bool ok = physical == MZGPU_FRONTIER_EMPTY ||
                (b->desc.upper != MZGPU_FRONTIER_EMPTY && b->desc.upper <= physical);
      if (!ok) break;
      pending.erase(pending.begin());
      // admission needs the exact length; release the slack of a loosely sized batch
      int32_t st = batch_resolve(b);
      if (st == MZGPU_OK) st = batch_shrink(b);
      if (st != MZGPU_OK && err == MZGPU_OK) err = st;
      insert_entry(b);
    }
  }
  // oldest first
  void all_batches(std::vector<mzgpu_batch*>& out) const {
    for (size_t i = merging.size(); i-- > 0;)
      for (auto* b : merging[i].batches) out.push_back(b);
    for (auto* b : pending) out.push_back(b);
  }
  ~mzgpu_spine() {
    for (auto& m : merging)
      for (auto* b : m.batches) mzgpu_batch_release(b);
    for (auto* b : pending) mzgpu_batch_release(b);
  }
};

static int32_t spine_take_err(mzgpu_spine* s) {
  int32_t e = s->err;
  s->err = MZGPU_OK;
  if (e == MZGPU_OK && s->ctx->sticky) e = s->ctx->sticky_code;
  return e;
}

extern "C" int32_t mzgpu_spine_new(mzgpu_ctx* ctx, uint32_t row_bytes, uint32_t effort,
                                   mzgpu_spine** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || !arrangement_row_bytes(row_bytes)) return MZGPU_E_INVALID;
  mzgpu_spine* s = new mzgpu_spine();
  s->ctx = ctx;
  s->rb = row_bytes;
  s->effort = effort ? effort : 1;
  *out = s;
  return MZGPU_OK;
}
extern "C" void mzgpu_spine_free(mzgpu_spine* s) { delete s; }
extern "C" int32_t mzgpu_spine_insert(mzgpu_spine* s, mzgpu_batch* batch) {
  if (s == nullptr || batch == nullptr || batch->rb != s->rb) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(s->ctx);
  if (batch->desc.lower == batch->desc.upper || batch->desc.lower != s->upper) {
    MZ_SET_ERR(s->ctx, "spine_insert: batch [%llu, %llu) does not extend trace upper %llu",
               (unsigned long long)batch->desc.lower, (unsigned long long)batch->desc.upper,
               (unsigned long long)s->upper);
    return MZGPU_E_FRONTIER;
  }
  mzgpu_batch_retain(batch);
  s->upper = batch->desc.upper;
  s->pending.push_back(batch);
  s->consider_merges();
  return spine_take_err(s);
}
extern "C" int32_t mzgpu_spine_exert(mzgpu_spine* s, uint64_t effort, int32_t* did_work) {
  if (s == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(s->ctx);
  if (did_work) *did_work = 0;
  s->tidy_layers();
  if (s->reduced()) return spine_take_err(s);
  bool any = false;
  for (auto& m : s->merging) any = any || m.has_merge;
  if (any) {
    // isize::try_from(effort).unwrap_or(isize::MAX) (trace.rs:1706)
    s->apply_fuel(effort > (uint64_t)INT64_MAX ? (long long)INT64_MAX : (long long)effort);
  } else {
    mzgpu_batch* e = nullptr;
    mzgpu_desc d = {s->upper, s->upper, s->since};
    MZ_TRY(make_empty_batch(s->ctx, s->rb, d, &e));
    s->introduce_batch(e, mzgpu_spine::level_of(effort));
  }
  if (did_work) *did_work = 1;
  return spine_take_err(s);
}
extern "C" uint64_t mzgpu_spine_exert_logic(const mzgpu_spine* s, uint32_t proportionality) {
  if (s == nullptr || proportionality == 0) return 0;
  uint32_t prop = proportionality;
  bool skipping = true, first = true;
  for (size_t i = s->merging.size(); i-- > 0;) {
    size_t count = s->merging[i].batches.size();
    u64 len = s->layer_len(s->merging[i]);
    if (skipping && count == 0) continue;
    skipping = false;
    if (count > 1) return 1000;
    if (!first && prop > 0 && len > 0) return 1000;
    first = false;
    prop /= 2;
  }
  return 0;
}
extern "C" int32_t mzgpu_spine_set_logical_compaction(mzgpu_spine* s, uint64_t f) {
  if (s == nullptr) return MZGPU_E_INVALID;
  if (f == MZGPU_FRONTIER_EMPTY || f > s->since) s->since = f;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_spine_set_physical_compaction(mzgpu_spine* s, uint64_t f) {
  if (s == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(s->ctx);
  if (f == MZGPU_FRONTIER_EMPTY || (s->physical != MZGPU_FRONTIER_EMPTY && f > s->physical)) s->physical = f;
  s->consider_merges();
  return spine_take_err(s);
}
extern "C" uint64_t mzgpu_spine_get_logical_compaction(const mzgpu_spine* s) { return s ? s->since : 0; }
extern "C" uint64_t mzgpu_spine_get_physical_compaction(const mzgpu_spine* s) {
  return s ? s->physical : 0;
}
extern "C" uint64_t mzgpu_spine_read_upper(const mzgpu_spine* s) { return s ? s->upper : 0; }

static void spine_through(mzgpu_spine* s, u64 through, std::vector<mzgpu_batch*>& out) {
  std::vector<mzgpu_batch*> all;
  s->all_batches(all);
  for (auto* b : all) {
    if (through == MZGPU_FRONTIER_EMPTY || (b->desc.upper != MZGPU_FRONTIER_EMPTY && b->desc.upper <= through))
      out.push_back(b);
  }
}
// the batches a reader of the arrangement probes: every batch, a merge still in flight on the side
// stream represented by its inputs
static void spine_readable(const mzgpu_spine* s, std::vector<mzgpu_batch*>& out) {
  std::vector<mzgpu_batch*> all;
  s->all_batches(all);
  for (auto* b : all) expand_readable(b, out);
}
extern "C" int32_t mzgpu_spine_batches_through(mzgpu_spine* s, uint64_t upper, mzgpu_batch** batches,
                                               uint32_t cap, uint32_t* n_out) {
  if (s == nullptr || n_out == nullptr) return MZGPU_E_INVALID;
  s->view.clear();
  spine_through(s, upper, s->view);
  *n_out = (uint32_t)s->view.size();
  if (s->view.size() > cap) return MZGPU_E_CAPACITY;
  for (size_t i = 0; i < s->view.size(); ++i) batches[i] = s->view[i];
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_spine_layers(const mzgpu_spine* s, uint64_t* out4, uint32_t cap_layers,
                                      uint32_t* n_layers) {
  if (s == nullptr || n_layers == nullptr) return MZGPU_E_INVALID;
  uint32_t n = 0;
  for (size_t i = s->merging.size(); i-- > 0;) {
    if (n >= cap_layers) return MZGPU_E_CAPACITY;
    auto& m = const_cast<mzgpu_spine*>(s)->merging[i];
    if (m.has_merge) mzgpu_spine::settle(m, true);
    out4[4 * n + 0] = m.batches.size();
    out4[4 * n + 1] = m.batches.size() > 0 ? blen(m.batches[0]) : 0;
    out4[4 * n + 2] = m.batches.size() > 1 ? blen(m.batches[1]) : 0;
    out4[4 * n + 3] = m.has_merge ? m.remaining : 0;
    ++n;
  }
  *n_layers = n;
  return MZGPU_OK;
}

// Device-visible view of a set of batches.  Batches still in flight are passed
// by their device header (length, mask), resolved ones by value.
static int32_t trace_view(mzgpu_ctx* ctx, const std::vector<mzgpu_batch*>& batches, TraceView* tv) {
  tv->n_batches = 0;
  for (auto* b : batches) {
    MZ_TRY(batch_ready(b));
    if (b->st.known && b->st.v[0] == 0) continue;
    if (tv->n_batches >= MZ_MAX_TRACE_BATCHES) {
      MZ_SET_ERR(ctx, "trace has more than %d non-empty batches", MZ_MAX_TRACE_BATCHES);
      return MZGPU_E_UNSUPPORTED;
    }
    BatchView& v = tv->b[tv->n_batches++];
    v.rows = b->rows.as<u64>();
    v.table = b->table.as<HashSlot>();
    if (b->st.known) {
      v.n = b->st.v[0];
      v.mask = b->st.v[1];
      v.hdr = nullptr;
    } else {
      v.n = 0;
      v.mask = 0;
      v.hdr = b->st.dptr();
    }
  }
  return MZGPU_OK;
}
// The view of every batch of a spine.
static int32_t trace_view_of(mzgpu_spine* s, TraceView* tv) {
  std::vector<mzgpu_batch*> batches;
  s->all_batches(batches);
  return trace_view(s->ctx, batches, tv);
}
// Upper bound on the matches of one probe row: the sum over batches of the
// longest key run.  *exact is false if some run length saturated.
static int32_t trace_fanout(const std::vector<mzgpu_batch*>& batches, u64* fan, bool* exact) {
  *fan = 0;
  *exact = true;
  for (auto* b : batches) {
    MZ_TRY(batch_resolve(b));
    if (b->st.v[0] == 0) continue;
    if (b->st.v[3] >= 1024) *exact = false;
    *fan += b->st.v[3];
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_spine_size(const mzgpu_spine* s, mzgpu_arrangement_size* out) {
  if (s == nullptr || out == nullptr) return MZGPU_E_INVALID;
  memset(out, 0, sizeof(*out));
  std::vector<mzgpu_batch*> all;
  s->all_batches(all);
  for (auto* b : all) {
    b->st.try_resolve();  // (never waits)
    const u64 len = b->st.known ? b->st.v[0] : b->len_ub;
    const u64 keys = b->st.known ? b->st.v[2] : 0;
    out->batches++;
    out->updates += len;
    out->size_bytes += len * b->rb + keys * sizeof(HashSlot);
    out->capacity_bytes += b->rows.bytes + b->table.bytes;
    out->allocations += (b->rows.p != nullptr ? 1 : 0) + (b->table.p != nullptr ? 1 : 0);
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_spine_export(mzgpu_spine* s, mzgpu_buf* out) {
  if (s == nullptr || out == nullptr || out->rb != s->rb) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(s->ctx);
  std::vector<mzgpu_batch*> all;
  s->all_batches(all);
  // fold the batches oldest-first with the merge kernel (advancing to `since`)
  DevMem acc;
  u64 acc_len = 0;
  MZ_TRY(acc.alloc(s->ctx, 16));
  for (auto* b : all) {
    DevMem m;
    u64 n = 0;
    MZ_TRY(batch_ready(b));
    MZ_TRY(batch_resolve(b));
    MZ_TRY(mz_merge_consolidate(s->ctx, s->rb, acc.p, acc_len, b->rows.p, b->st.v[0], s->since, &m, &n));
    acc = std::move(m);
    acc_len = n;
  }
  buf_adopt(out, std::move(acc), acc_len);
  return MZGPU_OK;
}

// ============================================================ join closures
// An MfpPlan closure of the probe operators (mzgpu_join_closure_new): the checked plan, and its copy in device
// memory that the probe kernels read (warp-uniform loads; the plan is too large for the kernel parameters).
struct mzgpu_join_closure {
  mzgpu_ctx* ctx;
  MfpDevPlan pl;
  DevMem dev;
  int out_rb() const { return (int)pl.plan.out_row_bytes; }
};
static int32_t mfp_build_plan(mzgpu_ctx* ctx, const mzgpu_mfp* plan, const mzgpu_mfp_map* map, uint32_t n_fn,
                              MfpDevPlan* out_pl);
extern "C" int32_t mzgpu_join_closure_new(mzgpu_ctx* ctx, const mzgpu_mfp* plan, const mzgpu_mfp_map* map,
                                          mzgpu_join_closure** out) {
  MZ_CHECK_CTX(ctx);
  if (plan == nullptr || out == nullptr) return MZGPU_E_INVALID;
  if (plan->in_row_bytes != 40) {
    MZ_SET_ERR(ctx, "join closure: the input is (key, stream value, lookup value), in_row_bytes 40, not %u",
               plan->in_row_bytes);
    return MZGPU_E_INVALID;
  }
  if (plan->n_temporal != 0) {
    MZ_SET_ERR(ctx, "join closure: %u temporal predicates (a JoinClosure's plan has none)", plan->n_temporal);
    return MZGPU_E_INVALID;
  }
  auto jc = std::unique_ptr<mzgpu_join_closure>(new mzgpu_join_closure());
  jc->ctx = ctx;
  MZ_TRY(mfp_build_plan(ctx, plan, map, 0, &jc->pl));
  MZ_TRY(jc->dev.alloc(ctx, sizeof(MfpDevPlan)));
  MZ_TRY(copy_in(ctx, jc->dev.p, &jc->pl, sizeof(MfpDevPlan), MZGPU_MEM_HOST));
  *out = jc.release();
  return MZGPU_OK;
}
extern "C" void mzgpu_join_closure_free(mzgpu_join_closure* jc) { delete jc; }

// The error rows of one call's probes with an MfpPlan closure: each probe leaves its raw rows as a chunk, and
// errs_flush appends them all to the caller's buffer, consolidated once.
struct ErrSink {
  struct Chunk {
    DevMem rows;
    Lazy4 len;
    u64 ub;
  };
  std::vector<Chunk> chunks;
};
// `n_out` set: the exact count of the appended rows is returned (join_core's fuel counts them)
static int32_t errs_flush(mzgpu_ctx* ctx, ErrSink& s, mzgpu_buf* errs, u64* n_out = nullptr) {
  if (n_out != nullptr) *n_out = 0;
  u64 ub = 0;
  for (auto& c : s.chunks) ub += c.ub;
  if (ub == 0) {
    s.chunks.clear();
    return MZGPU_OK;
  }
  mzgpu_buf all;
  const void* rows = s.chunks[0].rows.p;
  DLen n = dlen_of(s.chunks[0].len, 0);
  if (s.chunks.size() > 1) {
    all.ctx = ctx;
    all.rb = 32;
    all.len.set(ctx, 0);
    for (auto& c : s.chunks) MZ_TRY(buf_append_dev(&all, c.rows.p, dlen_of(c.len, 0), c.ub));
    rows = all.mem.p;
    n = buf_dlen(&all);
  }
  int32_t st;
  if (n_out == nullptr) {
    st = append_consolidated(ctx, 32, rows, n, ub, errs);
  } else {
    DevMem cons;
    u64 ccap = 0;
    Lazy4 clen;
    st = consolidate_dev(ctx, 32, rows, n, ub, &cons, &ccap, &clen);
    if (st == MZGPU_OK) st = clen.resolve();
    if (st == MZGPU_OK) {
      *n_out = clen.v[0];
      st = buf_append_dev(errs, cons.p, dlen_imm(*n_out), *n_out);
    }
  }
  s.chunks.clear();
  return st;
}
// A chunk of `cap` error rows with a zeroed device count, for a single-pass probe to fill.
static int32_t errs_chunk(mzgpu_ctx* ctx, const mzgpu_join_closure* jc, u64 cap, ErrSink* s, MfpProbe* mp) {
  s->chunks.emplace_back();
  ErrSink::Chunk& c = s->chunks.back();
  c.ub = cap;
  MZ_TRY(c.rows.alloc(ctx, cap * 32));
  MZ_TRY(c.len.make_pending(ctx));
  MZ_CUDA(ctx, cudaMemsetAsync(c.len.dptr(), 0, 8, ctx->stream));
  *mp = MfpProbe{(const MfpDevPlan*)jc->dev.p, jc->out_rb(), c.rows.as<u64>(), cap, c.len.dptr()};
  return MZGPU_OK;
}

// ================================================================ join_core
// The trace side of a probe, planned once for any stream: the view of the trace's batches (in the caller's
// storage: it is large), the kernel parameters, and the fan-out bound that decides the form a stream takes.
struct ProbePlan {
  TraceView* tv;
  ProbeParams pp;
  const mzgpu_join_closure* jc;  // an MfpPlan closure instead of pp's
  u64 fan;       // matches of one probe row at most: the sum over batches of the longest key run
  bool exact;    // no batch's longest run saturated
  u64 max_rows;  // the largest output bound the caller lets the bounded form take
  // n_ub probe rows yield at most n_ub x fan rows, and that bound is within the caller's limit
  bool within(u64 n_ub) const { return exact && fan > 0 && n_ub <= max_rows / fan; }
  // Bounded fan-out: one pass into a buffer of n_ub x fan rows -- the probe walks the trace once
  // instead of twice (count, write) and needs no read-back.  Otherwise the exact two-pass form runs.
  bool bounded(u64 n_ub) const { return within(n_ub) && mz_probe_tiles(n_ub, tv->n_batches) <= MZ_LB_TILES; }
  int rb() const { return jc != nullptr ? jc->out_rb() : pp.has_closure ? 32 : 40; }
};
// `mode` MZ_PROBE_HALF_LE / _LT or MZ_PROBE_JOIN.  Without a closure a half join writes (key, val2) -- the
// lookup value replaces the stream value -- and join_core the R40 row (key, val1, val2).  `jc` (an MfpPlan
// closure) takes the place of `closure`.
static int32_t probe_plan(mzgpu_ctx* ctx, const std::vector<mzgpu_batch*>& batches, int mode,
                          const mzgpu_closure* closure, u64 meet, bool swap_vals, u64 max_rows, TraceView* tv,
                          ProbePlan* p, const mzgpu_join_closure* jc = nullptr) {
  MZ_TRY(trace_fanout(batches, &p->fan, &p->exact));
  MZ_TRY(trace_view(ctx, batches, tv));
  p->tv = tv;
  p->max_rows = max_rows;
  p->jc = jc;
  memset(&p->pp, 0, sizeof(p->pp));
  p->pp.mode = mode;
  p->pp.meet = meet;
  p->pp.swap_vals = swap_vals ? 1 : 0;
  p->pp.has_closure = closure != nullptr || (mode != MZ_PROBE_JOIN && jc == nullptr) ? 1 : 0;
  if (jc == nullptr && closure != nullptr) {
    p->pp.closure = *closure;
  } else if (jc == nullptr && mode != MZ_PROBE_JOIN) {
    p->pp.closure.n_key_fields = 1;
    p->pp.closure.key_fields[0] = mzgpu_field{MZGPU_SRC_KEY, 0, 64, 0};
    p->pp.closure.n_val_fields = 1;
    p->pp.closure.val_fields[0] = mzgpu_field{MZGPU_SRC_VAL2, 0, 64, 0};
  }
  return MZGPU_OK;
}

// What becomes of a probe's output: appended to `out` as it is, appended consolidated, or consolidated and
// appended with its exact row count returned (join_core's fuel accounting reads it back anyway).
enum class ProbeOut { APPEND, APPEND_CONSOLIDATED, CONSOLIDATE_COUNT };
// A plan run over n stream rows (count possibly on the device, bound n_ub).  With an MfpPlan closure the error
// rows are left in `es`: the single-pass form gets room for one per match (n_ub x fan), so it cannot run out.
static int32_t probe_run(mzgpu_ctx* ctx, const ProbePlan& p, const u64* d_stream, DLen n, u64 n_ub, ProbeOut how,
                         mzgpu_buf* out, u64* n_out = nullptr, ErrSink* es = nullptr) {
  if (n_out != nullptr) *n_out = 0;
  if (n_ub == 0 || p.tv->n_batches == 0) return MZGPU_OK;
  const int rb = p.rb();
  DevMem res;
  Lazy4 rlen;
  DLen r_len;
  u64 r_ub = 0;
  MfpProbe mp;
  if (p.bounded(n_ub)) {
    const u64 bound = n_ub * p.fan;
    if (p.jc != nullptr) MZ_TRY(errs_chunk(ctx, p.jc, bound, es, &mp));
    const MfpProbe* mpp = p.jc != nullptr ? &mp : nullptr;
    if (how == ProbeOut::APPEND) {
      MZ_TRY(buf_reserve(out, out->ub + bound, true));
      Append a;
      MZ_TRY(buf_begin_append(out, &a));
      MZ_TRY(mz_probe_async(ctx, d_stream, n, n_ub, *p.tv, p.pp, out->mem.as<u64>(), a.base, out->cap, a.out_len,
                            mpp));
      buf_end_append(out, a, bound);
      if (mpp != nullptr) es->chunks.back().len.mark_written();
      return MZGPU_OK;
    }
    MZ_TRY(res.alloc(ctx, bound * rb));
    MZ_TRY(rlen.make_pending(ctx));
    MZ_TRY(mz_probe_async(ctx, d_stream, n, n_ub, *p.tv, p.pp, res.as<u64>(), dlen_imm(0), bound, rlen.dptr(), mpp));
    rlen.mark_written();
    if (mpp != nullptr) es->chunks.back().len.mark_written();
    if (how == ProbeOut::CONSOLIDATE_COUNT) MZ_TRY(rlen.resolve());
    r_len = dlen_of(rlen, 0);
    r_ub = rlen.known ? rlen.v[0] : bound;
  } else {
    u64 nn = 0;
    MZ_TRY(dlen_read(ctx, n, &nn));
    if (nn == 0) return MZGPU_OK;
    if (p.jc != nullptr) {
      mp = MfpProbe{(const MfpDevPlan*)p.jc->dev.p, rb, nullptr, 0, nullptr};
      es->chunks.emplace_back();
      ErrSink::Chunk& c = es->chunks.back();
      MZ_TRY(mz_probe(ctx, d_stream, nn, *p.tv, p.pp, &res, &r_ub, &mp, &c.rows, &c.ub));
      c.len.set(ctx, c.ub);
    } else {
      MZ_TRY(mz_probe(ctx, d_stream, nn, *p.tv, p.pp, &res, &r_ub));
    }
    r_len = dlen_imm(r_ub);
  }
  if (how == ProbeOut::APPEND) return buf_append_dev(out, res.p, r_len, r_ub);
  if (how == ProbeOut::APPEND_CONSOLIDATED) return append_consolidated(ctx, rb, res.p, r_len, r_ub, out);
  if (r_ub == 0) return MZGPU_OK;
  DevMem cons;
  u64 ccap = 0;
  Lazy4 clen;
  MZ_TRY(consolidate_dev(ctx, rb, res.p, r_len, r_ub, &cons, &ccap, &clen));
  MZ_TRY(clen.resolve());
  *n_out = clen.v[0];
  return buf_append_dev(out, cons.p, dlen_imm(*n_out), *n_out);
}

struct mzgpu_join {
  mzgpu_ctx* ctx;
  mzgpu_spine *t1, *t2;
  bool has_closure;
  mzgpu_closure closure;
  const mzgpu_join_closure* jc = nullptr;  // mzgpu_join_new_mfp (the caller keeps it alive)
  u64 ack1 = 0, ack2 = 0;
  struct Work {
    int side;
    mzgpu_batch* batch;
    std::vector<mzgpu_batch*> others;
    u64 cap;
    u64 pos = 0;  // rows of `batch` already joined (a work item is probed in slices)
  };
  std::deque<Work> todo;
  void release_work(Work& w) {
    mzgpu_batch_release(w.batch);
    for (auto* b : w.others) mzgpu_batch_release(b);
  }
  ~mzgpu_join() {
    for (auto& w : todo) release_work(w);
  }
};

static void join_enqueue(mzgpu_join* j, int side, mzgpu_batch* batch, u64 cap) {
  mzgpu_join::Work w;
  w.side = side;
  w.batch = batch;
  mzgpu_batch_retain(batch);
  {
    std::vector<mzgpu_batch*> through;
    spine_through(side == 0 ? j->t2 : j->t1, side == 0 ? j->ack2 : j->ack1, through);
    for (auto* b : through) expand_readable(b, w.others);
  }
  for (auto* b : w.others) mzgpu_batch_retain(b);
  w.cap = cap;
  j->todo.push_back(std::move(w));
}

static int32_t join_create(mzgpu_ctx* ctx, mzgpu_spine* trace1, mzgpu_spine* trace2, const mzgpu_closure* closure,
                           const mzgpu_join_closure* jc, mzgpu_join** out) {
  MZ_CHECK_CTX(ctx);
  if (trace1 == nullptr || trace2 == nullptr || out == nullptr || trace1->rb != 32 || trace2->rb != 32)
    return MZGPU_E_INVALID;
  MZ_TRY(validate_closure(ctx, closure));
  mzgpu_join* j = new mzgpu_join();
  j->ctx = ctx;
  j->jc = jc;
  j->t1 = trace1;
  j->t2 = trace2;
  j->has_closure = closure != nullptr;
  memset(&j->closure, 0, sizeof(j->closure));
  if (closure) j->closure = *closure;
  // pre-load (mz_join_core.rs:109-190): trace1's batches are acknowledged, then
  // each existing trace2 batch is joined against trace1 through ack1
  std::vector<mzgpu_batch*> all;
  trace1->all_batches(all);
  for (auto* b : all) j->ack1 = b->desc.upper;
  all.clear();
  trace2->all_batches(all);
  for (auto* b : all) {
    if (blen(b)) join_enqueue(j, 1, b, 0);
    j->ack2 = b->desc.upper;
  }
  *out = j;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_join_new(mzgpu_ctx* ctx, mzgpu_spine* trace1, mzgpu_spine* trace2,
                                  const mzgpu_closure* closure, mzgpu_join** out) {
  return join_create(ctx, trace1, trace2, closure, nullptr, out);
}
extern "C" int32_t mzgpu_join_new_mfp(mzgpu_ctx* ctx, mzgpu_spine* trace1, mzgpu_spine* trace2,
                                      const mzgpu_join_closure* jc, mzgpu_join** out) {
  MZ_CHECK_CTX(ctx);
  if (jc == nullptr || jc->ctx != ctx) return MZGPU_E_INVALID;
  return join_create(ctx, trace1, trace2, nullptr, jc, out);
}
extern "C" void mzgpu_join_free(mzgpu_join* j) { delete j; }

extern "C" int32_t mzgpu_join_core_push(mzgpu_join* j, int32_t side, mzgpu_batch* batch, uint64_t cap) {
  if (j == nullptr || batch == nullptr || (side != 0 && side != 1) || batch->rb != 32) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(j->ctx);
  u64& ack = side == 0 ? j->ack1 : j->ack2;
  if (ack <= batch->desc.lower) {
    if (blen(batch)) join_enqueue(j, side, batch, cap);
    ack = batch->desc.upper;
  }
  // physical compaction of both traces follows the acknowledged frontiers
  MZ_TRY(mzgpu_spine_set_physical_compaction(j->t1, j->ack1));
  MZ_TRY(mzgpu_spine_set_physical_compaction(j->t2, j->ack2));
  return MZGPU_OK;
}

// bulk probes (join_core work items): the bounded single-pass form may take this much output memory
#define MZ_BULK_BOUND_BYTES (12ull << 30)
static u64 mono_ns() {
  return (u64)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch())
      .count();
}
// rows of a work item's batch probed per slice: the reference's yield budget is 1M rows of work
// (linear_join.rs:145-151), so a bulk work item (hydration: 10M x 10M rows) yields ~10 times
#define MZ_JOIN_SLICE_ROWS (1ull << 20)
// Work::process; `errs` receives an MfpPlan closure's error rows, consolidated per slice, and they count as fuel
// (mz_join_core.rs:718-770 counts every result of the result function).
static int32_t join_work(mzgpu_join* j, uint64_t fuel_rows, uint64_t deadline_ns, mzgpu_buf* out, mzgpu_buf* errs,
                         int32_t* done) {
  const uint32_t out_rb = j->jc != nullptr ? (uint32_t)j->jc->out_rb() : j->has_closure ? 32 : 40;
  if (out->rb != out_rb) {
    MZ_SET_ERR(j->ctx, "join_core_work: output buffer row width %u, expected %u", out->rb, out_rb);
    return MZGPU_E_INVALID;
  }
  u64 produced = 0;
  // (at least one slice per call: a deadline that has already passed still makes progress)
  bool first = true;
  while (!j->todo.empty() && produced < fuel_rows && (first || deadline_ns == 0 || mono_ns() < deadline_ns)) {
    first = false;
    // the item leaves the queue only once its output has been appended: a failure below (more
    // batches than a trace view holds, counter arena, ...) leaves it queued, so no join work is lost
    mzgpu_join::Work& w = j->todo.front();
    for (auto* b : w.others) MZ_TRY(batch_resolve(b));
    MZ_TRY(batch_ready(w.batch));
    MZ_TRY(batch_resolve(w.batch));
    // this slice: rows [w.pos, w.pos + n_probe) of the work item's batch
    const u64 n_total = w.batch->st.v[0];
    // a caller that gave no deadline and has fuel left for more than one slice is not asking to be
    // yielded to: it gets slices as large as its fuel allows (up to 16M rows), which take the bulk
    // sort for the slice's output instead of ten 1M-row fused launches (BASELINE config 2)
    u64 slice = MZ_JOIN_SLICE_ROWS;
    if (deadline_ns == 0) slice = std::max<u64>(slice, std::min<u64>(fuel_rows - produced, 16ull << 20));
    const u64 n_probe = std::min<u64>(n_total - std::min(n_total, w.pos), slice);
    TraceView tv;
    ProbePlan plan;
    // (with an MfpPlan closure the bounded form also holds one error row per match)
    MZ_TRY(probe_plan(j->ctx, w.others, MZ_PROBE_JOIN, j->has_closure ? &j->closure : nullptr, w.cap, w.side == 1,
                      MZ_BULK_BOUND_BYTES / (out_rb + (j->jc != nullptr ? 32 : 0)), &tv, &plan, j->jc));
    // Work::process consolidates each work item's output buffer before sending
    u64 n_cons = 0, n_errs = 0;
    ErrSink es;
    MZ_TRY(probe_run(j->ctx, plan, w.batch->rows.as<u64>() + w.pos * 4, dlen_imm(n_probe), n_probe,
                     ProbeOut::CONSOLIDATE_COUNT, out, &n_cons, &es));
    if (j->jc != nullptr) MZ_TRY(errs_flush(j->ctx, es, errs, &n_errs));
    w.pos += n_probe;
    if (w.pos >= n_total) {
      j->release_work(w);
      j->todo.pop_front();
    }
    produced += n_cons + n_errs;
    j->ctx->stats.rows_out += n_cons;
  }
  if (done) *done = j->todo.empty() ? 1 : 0;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_join_core_work_until(mzgpu_join* j, uint64_t fuel_rows, uint64_t deadline_ns,
                                              mzgpu_buf* out, int32_t* done) {
  if (j == nullptr || out == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(j->ctx);
  if (j->jc != nullptr) {
    MZ_SET_ERR(j->ctx, "join_core_work: a join with an MfpPlan closure works through mzgpu_join_core_work_mfp");
    return MZGPU_E_INVALID;
  }
  return join_work(j, fuel_rows, deadline_ns, out, nullptr, done);
}
extern "C" int32_t mzgpu_join_core_work_mfp(mzgpu_join* j, uint64_t fuel_rows, uint64_t deadline_ns, mzgpu_buf* out,
                                            mzgpu_buf* errs, int32_t* done) {
  if (j == nullptr || out == nullptr || errs == nullptr || j->jc == nullptr || errs->rb != 32 || errs == out)
    return MZGPU_E_INVALID;
  MZ_CHECK_CTX(j->ctx);
  return join_work(j, fuel_rows, deadline_ns, out, errs, done);
}
extern "C" int32_t mzgpu_join_core_work(mzgpu_join* j, uint64_t fuel_rows, mzgpu_buf* out, int32_t* done) {
  return mzgpu_join_core_work_until(j, fuel_rows, 0, out, done);
}

// ================================================================ half_join
// half joins: the bounded single-pass form may take this many output rows; beyond it (heavy skew) the
// exact two-pass form runs
#define MZ_BOUND_MAX_ROWS (48ull << 20)

// One half join: a stream probes a trace, the results are appended to `out`.
struct HalfJoinReq {
  mzgpu_buf* stream;  // the stream to probe with, or ...
  mzgpu_spine* trace;
  int32_t cmp_mode;
  const mzgpu_closure* closure;
  mzgpu_buf* out;
  // ... a sealed batch whose update stream (build_update_stream: rows at `skip_time` dropped,
  // `pre` applied) is formed inside the probe kernel
  mzgpu_batch* src = nullptr;
  const mzgpu_closure* pre = nullptr;
  u64 skip_time = MZGPU_FRONTIER_EMPTY;
  const mzgpu_join_closure* jc = nullptr;  // an MfpPlan closure in place of `closure`
};
static uint32_t req_out_rb(const HalfJoinReq& r) { return r.jc != nullptr ? (uint32_t)r.jc->out_rb() : 32; }
static const u64* req_rows(const HalfJoinReq& r) { return r.src ? r.src->rows.as<u64>() : r.stream->mem.as<u64>(); }
static DLen req_dlen(const HalfJoinReq& r) { return r.src ? batch_dlen(r.src) : buf_dlen(r.stream); }
static u64 req_ub(const HalfJoinReq& r) { return r.src ? r.src->len_ub : r.stream->ub; }
// a source batch of 32-byte rows, or a buffer of them other than the output
static bool req_stream_ok(const HalfJoinReq& r) {
  return r.src != nullptr ? r.src->rb == 32 : r.stream != nullptr && r.stream != r.out && r.stream->rb == 32;
}
// The argument check every half-join entry point makes of each request; `stream_ok` is its check of the rows
// the request probes with.  Refusals set no message; a malformed closure sets its own.
static int32_t half_join_check(mzgpu_ctx* ctx, bool stream_ok, const HalfJoinReq& r) {
  if (!stream_ok || r.trace == nullptr || r.out == nullptr || r.trace->rb != 32 || r.out->rb != req_out_rb(r) ||
      (r.cmp_mode != MZGPU_HALFJOIN_LE && r.cmp_mode != MZGPU_HALFJOIN_LT) || (r.jc != nullptr && r.jc->ctx != ctx))
    return MZGPU_E_INVALID;
  MZ_TRY(validate_closure(ctx, r.pre));
  return validate_closure(ctx, r.closure);
}
static int32_t half_join_plan(mzgpu_ctx* ctx, const HalfJoinReq& r, TraceView* tv, ProbePlan* p) {
  std::vector<mzgpu_batch*> all;
  spine_readable(r.trace, all);
  // with an MfpPlan closure the bounded form also holds one 32-byte error row per match: the same bytes in all
  const u64 max_rows = r.jc != nullptr ? MZ_BOUND_MAX_ROWS * 32 / (r.jc->out_rb() + 32) : MZ_BOUND_MAX_ROWS;
  return probe_plan(ctx, all, r.cmp_mode == MZGPU_HALFJOIN_LE ? MZ_PROBE_HALF_LE : MZ_PROBE_HALF_LT, r.closure, 0,
                    false, max_rows, tv, p, r.jc);
}
static int32_t half_join_dev(mzgpu_ctx* ctx, const HalfJoinReq& r, const u64* d_stream, DLen n, u64 n_ub,
                             int32_t consolidate_output, ErrSink* es = nullptr) {
  if (n_ub == 0) return MZGPU_OK;
  TraceView tv;
  ProbePlan plan;
  MZ_TRY(half_join_plan(ctx, r, &tv, &plan));
  return probe_run(ctx, plan, d_stream, n, n_ub, consolidate_output ? ProbeOut::APPEND_CONSOLIDATED : ProbeOut::APPEND,
                   r.out, nullptr, es);
}
// the error buffer of an MfpPlan closure's half joins: R32, apart from every stream and output
static bool errs_ok(const mzgpu_buf* errs, const mzgpu_buf* stream, const mzgpu_buf* out) {
  return errs != nullptr && errs->rb == 32 && errs != stream && errs != out;
}

extern "C" int32_t mzgpu_half_join(mzgpu_ctx* ctx, const mzgpu_r32* stream, uint64_t n, int32_t mem,
                                   mzgpu_spine* trace, int32_t cmp_mode, const mzgpu_closure* closure,
                                   int32_t consolidate_output, mzgpu_buf* out) {
  MZ_CHECK_CTX(ctx);
  const HalfJoinReq r{nullptr, trace, cmp_mode, closure, out};
  MZ_TRY(half_join_check(ctx, stream != nullptr || n == 0, r));
  DevMem in;
  const u64* d_stream;
  MZ_TRY(entry_rows_in(ctx, stream, n, mem, 32, &in, &d_stream));
  return half_join_dev(ctx, r, d_stream, dlen_imm(n), n, consolidate_output);
}
extern "C" int32_t mzgpu_half_join_buf(mzgpu_ctx* ctx, mzgpu_buf* stream, mzgpu_spine* trace, int32_t cmp_mode,
                                       const mzgpu_closure* closure, int32_t consolidate_output, mzgpu_buf* out) {
  MZ_CHECK_CTX(ctx);
  const HalfJoinReq r{stream, trace, cmp_mode, closure, out};
  MZ_TRY(half_join_check(ctx, req_stream_ok(r), r));
  ctx->stats.rows_in += stream->ub;
  return half_join_dev(ctx, r, stream->mem.as<u64>(), buf_dlen(stream), stream->ub, consolidate_output);
}
extern "C" int32_t mzgpu_half_join_mfp(mzgpu_ctx* ctx, const mzgpu_r32* stream, uint64_t n, int32_t mem,
                                       mzgpu_spine* trace, int32_t cmp_mode, const mzgpu_join_closure* jc,
                                       int32_t consolidate_output, mzgpu_buf* out, mzgpu_buf* errs) {
  MZ_CHECK_CTX(ctx);
  HalfJoinReq r{nullptr, trace, cmp_mode, nullptr, out};
  r.jc = jc;
  if (jc == nullptr || !errs_ok(errs, nullptr, out)) return MZGPU_E_INVALID;
  MZ_TRY(half_join_check(ctx, stream != nullptr || n == 0, r));
  DevMem in;
  const u64* d_stream;
  MZ_TRY(entry_rows_in(ctx, stream, n, mem, 32, &in, &d_stream));
  ErrSink es;
  MZ_TRY(half_join_dev(ctx, r, d_stream, dlen_imm(n), n, consolidate_output, &es));
  return errs_flush(ctx, es, errs);
}
extern "C" int32_t mzgpu_half_join_mfp_buf(mzgpu_ctx* ctx, mzgpu_buf* stream, mzgpu_spine* trace, int32_t cmp_mode,
                                           const mzgpu_join_closure* jc, int32_t consolidate_output, mzgpu_buf* out,
                                           mzgpu_buf* errs) {
  MZ_CHECK_CTX(ctx);
  HalfJoinReq r{stream, trace, cmp_mode, nullptr, out};
  r.jc = jc;
  if (jc == nullptr || !errs_ok(errs, stream, out)) return MZGPU_E_INVALID;
  MZ_TRY(half_join_check(ctx, req_stream_ok(r), r));
  ctx->stats.rows_in += stream->ub;
  ErrSink es;
  MZ_TRY(half_join_dev(ctx, r, stream->mem.as<u64>(), buf_dlen(stream), stream->ub, consolidate_output, &es));
  return errs_flush(ctx, es, errs);
}

static int32_t map_rows_into(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const mzgpu_closure* closure,
                             u64 skip_time, mzgpu_buf* out);
// k <= MZ_PROBE_MANY_MAX half joins in one launch (mz_probe_async_many).  Requests whose output buffers
// coincide must be adjacent: they form a chain whose results are appended in request order -- the last stage
// of the delta paths, whose outputs are concatenated (delta_join.rs:302-308).  Anything the single launch
// cannot take (unbounded fan-out, an empty stream or trace, a buffer named twice apart) runs request by
// request; the results are the same either way.
static int32_t half_join_many_dev(mzgpu_ctx* ctx, int k, const HalfJoinReq* reqs, ErrSink* es) {
  static thread_local TraceView tvs[MZ_PROBE_MANY_MAX];  // large: kept off the stack
  ProbePlan plans[MZ_PROBE_MANY_MAX];
  int planned = 0;  // requests [0, planned) have their trace side planned
  auto one_by_one = [&]() -> int32_t {
    for (int j = 0; j < k; ++j) {
      const HalfJoinReq& r = reqs[j];
      mzgpu_buf tmp;
      const mzgpu_buf* s = r.stream;
      if (r.src != nullptr) {
        // the separate operators: update stream into a scratch buffer, then the half join
        tmp.ctx = ctx;
        tmp.rb = 32;
        tmp.len.set(ctx, 0);
        MZ_TRY(map_rows_into(ctx, req_rows(r), req_dlen(r), req_ub(r), r.pre, r.skip_time, &tmp));
        s = &tmp;
      }
      // the stream is read now, not when the chain was planned: it may be an earlier request's output
      if (s->ub == 0) continue;
      // nothing between planning and running changes a spine: the chain's plan of this trace still holds
      if (j >= planned) MZ_TRY(half_join_plan(ctx, r, &tvs[j], &plans[j]));
      MZ_TRY(probe_run(ctx, plans[j], s->mem.as<u64>(), buf_dlen(s), s->ub, ProbeOut::APPEND, r.out, nullptr, es));
    }
    return MZGPU_OK;
  };
  for (int j = 0; j < k; ++j)
    if (reqs[j].src != nullptr) MZ_TRY(batch_ready(reqs[j].src));
  bool any_src = false;
  for (int j = 0; j < k; ++j) any_src = any_src || reqs[j].src != nullptr;
  if (k < 2 && !any_src) return one_by_one();
  u64 tiles = 0;
  for (int j = 0; j < k; ++j) {
    const HalfJoinReq& r = reqs[j];
    for (int i = 0; i + 1 < j; ++i)
      if (reqs[i].out == r.out && reqs[j - 1].out != r.out) return one_by_one();
    for (int i = 0; i < k; ++i)
      if (reqs[i].stream != nullptr && reqs[i].stream == r.out) return one_by_one();
    if (req_ub(r) == 0 || req_out_rb(r) != req_out_rb(reqs[0])) return one_by_one();
    MZ_TRY(half_join_plan(ctx, r, &tvs[j], &plans[j]));
    planned = j + 1;
    if (tvs[j].n_batches == 0 || !plans[j].within(req_ub(r))) return one_by_one();
    tiles += mz_probe_tiles(req_ub(r), tvs[j].n_batches);
  }
  // the requests share the look-back state: their tiles together must fit
  if (tiles > MZ_LB_TILES) return one_by_one();
  // chains: reserve each output for the sum of its requests' bounds, open one append per chain
  ProbeJobHost jobs[MZ_PROBE_MANY_MAX];
  Append app[MZ_PROBE_MANY_MAX];
  u64 chain_bound[MZ_PROBE_MANY_MAX] = {};
  MfpProbe mps[MZ_PROBE_MANY_MAX];
  mzgpu_buf* chain_out[MZ_PROBE_MANY_MAX];
  int nc = 0;
  for (int j = 0; j < k; ++j) {
    if (j == 0 || reqs[j].out != reqs[j - 1].out) chain_out[nc++] = reqs[j].out;
    jobs[j].chain = nc - 1;
    chain_bound[nc - 1] += req_ub(reqs[j]) * plans[j].fan;
  }
  // MfpPlan closures: one error chunk for the launch, room for one error row per match of every request
  const bool mfp = reqs[0].jc != nullptr;
  if (mfp) {
    u64 err_cap = 0;
    for (int c = 0; c < nc; ++c) err_cap += chain_bound[c];
    MZ_TRY(errs_chunk(ctx, reqs[0].jc, err_cap, es, &mps[0]));
    for (int j = 0; j < k; ++j) {
      mps[j] = mps[0];
      mps[j].pl = (const MfpDevPlan*)reqs[j].jc->dev.p;
    }
  }
  for (int c = 0; c < nc; ++c) {
    MZ_TRY(buf_reserve(chain_out[c], chain_out[c]->ub + chain_bound[c], true));
    MZ_TRY(buf_begin_append(chain_out[c], &app[c]));
  }
  for (int j = 0; j < k; ++j) {
    const int c = jobs[j].chain;
    jobs[j].d_stream = req_rows(reqs[j]);
    jobs[j].n = req_dlen(reqs[j]);
    jobs[j].n_ub = req_ub(reqs[j]);
    jobs[j].has_pre = reqs[j].src != nullptr;
    jobs[j].pre = reqs[j].pre;
    jobs[j].skip_time = reqs[j].skip_time;
    jobs[j].trace = &tvs[j];
    jobs[j].pp = &plans[j].pp;
    jobs[j].d_out = chain_out[c]->mem.as<u64>();
    jobs[j].out_base = app[c].base;
    jobs[j].out_cap = chain_out[c]->cap;
    jobs[j].d_out_len = app[c].out_len;
    jobs[j].mfp = mfp ? &mps[j] : nullptr;
  }
  MZ_TRY(mz_probe_async_many(ctx, k, jobs));
  for (int cc = 0; cc < nc; ++cc) buf_end_append(chain_out[cc], app[cc], chain_bound[cc]);
  if (mfp) es->chunks.back().len.mark_written();
  return MZGPU_OK;
}
// The *_many entry points: request j is built by req(j), checked and its rows counted before request j + 1 is
// checked; then groups of at most MZ_PROBE_MANY_MAX run, never splitting a chain's adjacency.
// With MfpPlan closures (`errs` set) the errors of all the requests are appended to `errs`, consolidated once.
template <class Req>
static int32_t half_join_many_entry(mzgpu_ctx* ctx, uint32_t k, bool arrays_ok, Req req, mzgpu_buf* errs = nullptr) {
  MZ_CHECK_CTX(ctx);
  if (k == 0) return MZGPU_OK;
  if (!arrays_ok || k > 64) return MZGPU_E_INVALID;
  ErrSink es;
  std::vector<HalfJoinReq> reqs(k);
  for (uint32_t j = 0; j < k; ++j) {
    reqs[j] = req(j);
    if (errs != nullptr && (reqs[j].jc == nullptr || !errs_ok(errs, reqs[j].stream, reqs[j].out)))
      return MZGPU_E_INVALID;
    MZ_TRY(half_join_check(ctx, req_stream_ok(reqs[j]), reqs[j]));
    ctx->stats.rows_in += req_ub(reqs[j]);
  }
  for (uint32_t at = 0; at < k; at += MZ_PROBE_MANY_MAX)
    MZ_TRY(half_join_many_dev(ctx, (int)std::min<uint32_t>(MZ_PROBE_MANY_MAX, k - at), reqs.data() + at, &es));
  return errs != nullptr ? errs_flush(ctx, es, errs) : MZGPU_OK;
}
extern "C" int32_t mzgpu_half_join_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf* const* streams,
                                        mzgpu_spine* const* traces, const int32_t* cmp_modes,
                                        const mzgpu_closure* const* closures, mzgpu_buf* const* outs) {
  const bool arrays_ok = streams != nullptr && traces != nullptr && cmp_modes != nullptr && outs != nullptr;
  return half_join_many_entry(ctx, k, arrays_ok, [&](uint32_t j) {
    return HalfJoinReq{streams[j], traces[j], cmp_modes[j], closures ? closures[j] : nullptr, outs[j]};
  });
}
extern "C" int32_t mzgpu_half_join_many_mfp(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf* const* streams,
                                            mzgpu_spine* const* traces, const int32_t* cmp_modes,
                                            const mzgpu_join_closure* const* jcs, mzgpu_buf* const* outs,
                                            mzgpu_buf* errs) {
  const bool arrays_ok = streams != nullptr && traces != nullptr && cmp_modes != nullptr && jcs != nullptr &&
                         outs != nullptr && errs != nullptr;
  return half_join_many_entry(
      ctx, k, arrays_ok,
      [&](uint32_t j) {
        HalfJoinReq r{streams[j], traces[j], cmp_modes[j], nullptr, outs[j]};
        r.jc = jcs[j];
        return r;
      },
      errs);
}
extern "C" int32_t mzgpu_delta_first_stage_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_batch* const* batches,
                                                const mzgpu_closure* const* initial_closures,
                                                const uint64_t* skip_times, mzgpu_spine* const* traces,
                                                const int32_t* cmp_modes, const mzgpu_closure* const* closures,
                                                mzgpu_buf* const* outs) {
  const bool arrays_ok = batches != nullptr && skip_times != nullptr && traces != nullptr && cmp_modes != nullptr &&
                         outs != nullptr;
  return half_join_many_entry(ctx, k, arrays_ok, [&](uint32_t j) {
    return HalfJoinReq{nullptr, traces[j], cmp_modes[j], closures ? closures[j] : nullptr, outs[j], batches[j],
                       initial_closures ? initial_closures[j] : nullptr, skip_times[j]};
  });
}

// rows -> closure(rows) appended to `out`; at most one output row per input row
static int32_t map_rows_into(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const mzgpu_closure* closure,
                             u64 skip_time, mzgpu_buf* out) {
  if (n_ub == 0) return MZGPU_OK;
  if ((n_ub + 255) / 256 > MZ_LB_TILES) {
    u64 nn = 0;
    MZ_TRY(dlen_read(ctx, n, &nn));
    DevMem res;
    u64 n_res = 0;
    MZ_TRY(mz_map_rows_dev(ctx, d_rows, nn, closure, skip_time, &res, &n_res));
    return buf_append_dev(out, res.p, dlen_imm(n_res), n_res);
  }
  MZ_TRY(buf_reserve(out, out->ub + n_ub, true));
  Append a;
  MZ_TRY(buf_begin_append(out, &a));
  MZ_TRY(mz_map_rows_async(ctx, d_rows, n, n_ub, closure, skip_time, out->mem.as<u64>(), a.base, out->cap,
                           a.out_len));
  buf_end_append(out, a, n_ub);
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_update_stream(mzgpu_ctx* ctx, mzgpu_batch* batch,
                                       const mzgpu_closure* initial_closure, uint64_t skip_time,
                                       mzgpu_buf* out) {
  MZ_CHECK_CTX(ctx);
  if (batch == nullptr || out == nullptr || batch->rb != 32 || out->rb != 32) return MZGPU_E_INVALID;
  MZ_TRY(validate_closure(ctx, initial_closure));
  MZ_TRY(batch_ready(batch));
  return map_rows_into(ctx, batch->rows.as<u64>(), batch_dlen(batch), batch->len_ub, initial_closure, skip_time,
                       out);
}

extern "C" int32_t mzgpu_map_rows(mzgpu_ctx* ctx, const mzgpu_r32* rows, uint64_t n, int32_t mem,
                                  const mzgpu_closure* closure, mzgpu_buf* out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || (rows == nullptr && n) || out->rb != 32) return MZGPU_E_INVALID;
  MZ_TRY(validate_closure(ctx, closure));
  if (n == 0) return MZGPU_OK;
  DevMem in;
  const u64* d_rows = (const u64*)rows;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(in.alloc(ctx, n * 32));
    MZ_TRY(copy_in(ctx, in.p, rows, n * 32, mem));
    d_rows = in.as<u64>();
  }
  return map_rows_into(ctx, d_rows, dlen_imm(n), n, closure, MZGPU_FRONTIER_EMPTY, out);
}

// =================================================================== reduce
// Which operator a mzgpu_reduce is; each pair of step entry points takes one shape.
enum class ReduceShape {
  ACCUM,           // mzgpu_reduce_new and mzgpu_topk_new, told apart by agg_kind
  LANES,           // mzgpu_reduce_lanes_new[_having]
  MONOTONIC,       // mzgpu_reduce_monotonic_new
  HIERARCHICAL,    // mzgpu_reduce_hierarchical_new
  TOPK_MONOTONIC,  // mzgpu_topk_monotonic_new
  TOPK_BASIC,      // mzgpu_topk_basic_new
};
struct mzgpu_reduce {
  mzgpu_ctx* ctx;
  ReduceShape shape;
  // LANES: the lane class (1, 2, 4, 8); MONOTONIC / HIERARCHICAL: the mono class (4, 8)
  int cls = 0;
  mzgpu_batcher* batcher = nullptr;
  mzgpu_spine* input = nullptr;
  // ACCUM: the aggregate kind, and mzgpu_topk_new's parameters.  LANES: the first lane's kind without the
  // DISTINCT bit, which class 1 runs the one-column kernels with.
  int agg_kind = 0;
  TopKParams topk = {-1, 0, 0};
  // LANES, MONOTONIC, HIERARCHICAL: the lane descriptors
  LaneSet lanes = {};
  // LANES: the distinct lanes (MZGPU_ACCUM_DISTINCT), in lane order: the lane index, and the batcher and R32
  // pair arrangement of its (key, value) pairs
  int n_distinct = 0;
  u32 distinct_lane[MZGPU_MAX_ACCUM_LANES] = {};
  mzgpu_batcher* pair_batcher[MZGPU_MAX_ACCUM_LANES] = {};
  mzgpu_spine* pairs[MZGPU_MAX_ACCUM_LANES] = {};
  // LANES from mzgpu_reduce_lanes_new_having: the validated HAVING program, run by the corrections kernels
  bool has_having = false;
  mzgpu_having having = {};
  // MONOTONIC, HIERARCHICAL: the lanes' encodings and the value bits they read
  MonoXor mono = {};
  u64 mono_mask[2] = {0, 0};
  // MONOTONIC, TOPK_MONOTONIC: consolidate_named_if's flag
  bool must_consolidate = false;
  // TOPK_MONOTONIC, TOPK_BASIC: the order lanes and limit
  TopKOrder tko = {};
  // TOPK_BASIC: the offset (clamped to INT64_MAX), and the batcher and R32 arrangement of the negatives,
  // (key, 0, time, change in the key's negative-count rows)
  i64 topk_offset = 0;
  mzgpu_batcher* neg_batcher = nullptr;
  mzgpu_spine* negs = nullptr;
  int32_t failed = MZGPU_OK;  // set when an activation failed after its seal (reduce_dev)
  std::string failed_msg;
  ~mzgpu_reduce() {
    delete batcher;
    delete input;
    delete neg_batcher;
    delete negs;
    for (int j = 0; j < n_distinct; ++j) {
      delete pair_batcher[j];
      delete pairs[j];
    }
  }
};

// A new operator of `shape` with its input batcher and arrangement of arr_rb-byte rows.
static int32_t reduce_alloc(mzgpu_ctx* ctx, ReduceShape shape, uint32_t arr_rb, std::unique_ptr<mzgpu_reduce>* out) {
  std::unique_ptr<mzgpu_reduce> r(new mzgpu_reduce());
  r->ctx = ctx;
  r->shape = shape;
  MZ_TRY(mzgpu_batcher_new(ctx, arr_rb, &r->batcher));
  MZ_TRY(mzgpu_spine_new(ctx, arr_rb, 1, &r->input));
  *out = std::move(r);
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_reduce_new(mzgpu_ctx* ctx, int32_t agg_kind, mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || agg_kind < MZGPU_AGG_COUNT_SUM_I64 || agg_kind > MZGPU_AGG_MAX) return MZGPU_E_INVALID;
  // accumulable kinds arrange exploded diffs (RACC); MIN/MAX arranges the (key, value) rows themselves
  const uint32_t rb = (agg_kind == MZGPU_AGG_MIN || agg_kind == MZGPU_AGG_MAX) ? 32 : 80;
  std::unique_ptr<mzgpu_reduce> r;
  MZ_TRY(reduce_alloc(ctx, ReduceShape::ACCUM, rb, &r));
  r->agg_kind = agg_kind;
  *out = r.release();
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_topk_new(mzgpu_ctx* ctx, int64_t limit, uint64_t offset, int32_t descending,
                                  mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr) return MZGPU_E_INVALID;
  std::unique_ptr<mzgpu_reduce> r;
  MZ_TRY(reduce_alloc(ctx, ReduceShape::ACCUM, 32, &r));
  r->agg_kind = MZGPU_AGG_TOPK;
  r->topk.limit = limit < 0 ? -1 : limit;
  r->topk.offset = offset;
  r->topk.descending = descending != 0;
  *out = r.release();
  return MZGPU_OK;
}
extern "C" void mzgpu_reduce_free(mzgpu_reduce* r) { delete r; }
extern "C" mzgpu_spine* mzgpu_reduce_input_trace(mzgpu_reduce* r) { return r ? r->input : nullptr; }

// The distinct lanes' part of an activation (build_accumulable's distinct_aggrs, reduce.rs:1338-1373): the
// input's (key, value) pairs of every distinct lane (one launch), the pair batchers sealed at `upper` (shared
// cooperative launches), and the presence changes of the new pair batches (one launch) pushed into the main
// batcher as one more stash segment.  pair_new receives the sealed pair batches (the caller inserts them);
// *sealed is set once the pair batchers' frontiers may have moved.
static int32_t distinct_step(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper,
                             mzgpu_batch** pair_new, bool* sealed) {
  mzgpu_ctx* ctx = r->ctx;
  const int d = r->n_distinct;
  if (n_ub) {
    Seg segs[MZGPU_MAX_ACCUM_LANES];
    u64* outs[MZGPU_MAX_ACCUM_LANES] = {};
    u64* lens[MZGPU_MAX_ACCUM_LANES] = {};
    for (int j = 0; j < d; ++j) {
      MZ_TRY(segs[j].rows.alloc(ctx, n_ub * 32));
      outs[j] = segs[j].rows.as<u64>();
      if (n.p == nullptr) {
        segs[j].len.set(ctx, n.imm);
      } else {
        MZ_TRY(segs[j].len.make_pending(ctx));
        lens[j] = segs[j].len.dptr();
      }
      segs[j].ub = n.p == nullptr ? n.imm : n_ub;
    }
    MZ_TRY(mz_distinct_pairs(ctx, d_rows, n, n_ub, r->lanes, outs, lens));
    for (int j = 0; j < d; ++j) {
      if (n.p != nullptr) segs[j].len.mark_written();
      MZ_TRY(batcher_push_seg(r->pair_batcher[j], std::move(segs[j])));
    }
  }
  *sealed = true;
  MZ_TRY(batcher_seal_many(d, r->pair_batcher, upper, pair_new));
  std::vector<TraceView> tvs((size_t)d);
  std::vector<mzgpu_batch*> prior;
  DistinctJobHost jobs[MZGPU_MAX_ACCUM_LANES];
  u64 cap = 0;
  for (int j = 0; j < d; ++j) {
    prior.clear();
    r->pairs[j]->all_batches(prior);
    MZ_TRY(trace_view(ctx, prior, &tvs[(size_t)j]));
    const mzgpu_batch* b = pair_new[j];
    jobs[j] = DistinctJobHost{b->rows.as<u64>(), batch_dlen(b), b->len_ub, r->distinct_lane[j], &tvs[(size_t)j]};
    cap += b->len_ub;
  }
  if (cap == 0) return MZGPU_OK;
  // at most one presence change per new pair row
  Seg s;
  MZ_TRY(s.rows.alloc(ctx, cap * mz_lane_arr_bytes(r->cls)));
  MZ_TRY(mz_distinct_presence(ctx, r->cls, d, jobs, s.rows.as<u64>(), cap, &s.len, &s.word));
  s.ub = cap;
  return batcher_push_seg(r->batcher, std::move(s));
}

// The start of every reduce activation.  An earlier activation that lost its corrections left the operator
// dead (not the worker): it reports that status.  Batches sealed by earlier activations are merge-eligible
// now; their lengths have reached the host with whatever the caller read since (no extra wait).
static int32_t reduce_begin(mzgpu_reduce* r) {
  if (r->failed != MZGPU_OK) {
    r->ctx->last_error = r->failed_msg;
    return r->failed;
  }
  return mzgpu_spine_set_physical_compaction(r->input, r->input->upper);
}

// A failure once an activation has sealed a batch means its corrections are missing from the output, which
// no later activation can repair: the operator reports the first such status from now on (a sticky context
// reports its own).
static int32_t reduce_kill_on_failure(mzgpu_reduce* r, int32_t st) {
  if (st != MZGPU_OK && !r->ctx->sticky && r->failed == MZGPU_OK) {
    r->failed = st;
    r->failed_msg = r->ctx->last_error;
  }
  return st;
}

// A sealed batch joins its trace whatever happened since the seal (the seal consumed the batcher's rows and
// advanced its frontier, and the arrangement stays consistent with that frontier); returns the insert's status.
static int32_t trace_join(mzgpu_spine* trace, mzgpu_batch* batch) {
  int32_t ins = MZGPU_OK;
  if (batch->desc.lower != batch->desc.upper) ins = mzgpu_spine_insert(trace, batch);
  mzgpu_batch_release(batch);
  return ins;
}

// The end of an activation after its seal: the batch joins the input trace, then the kill rule on the first
// failure of the two.
static int32_t reduce_seal_tail(mzgpu_reduce* r, mzgpu_batch* batch, int32_t st) {
  const int32_t ins = trace_join(r->input, batch);
  return reduce_kill_on_failure(r, st != MZGPU_OK ? st : ins);
}

// The single-pass (look-back) form of the correction kernels covers a batch of n rows with at most per_row
// output rows each when its tiles fit the look-back state and its output fits MZ_BOUND_MAX_ROWS.
static bool single_pass_fits(u64 n, u64 per_row) {
  return (n + 255) / 256 <= MZ_LB_TILES && per_row * n <= MZ_BOUND_MAX_ROWS;
}

// A segment of the input's length: the same count as the input rows, shared with nothing (a device-resident
// count is copied on the device).
static int32_t seg_len_of_input(mzgpu_ctx* ctx, DLen n, u64 n_ub, Seg* s) {
  if (n.p == nullptr) {
    s->len.set(ctx, n.imm);
    s->ub = n.imm;
    return MZGPU_OK;
  }
  MZ_TRY(s->len.make_pending(ctx));
  MZ_CUDA(ctx, cudaMemcpyAsync(s->len.dptr(), n.p, 8, cudaMemcpyDeviceToDevice, ctx->stream));
  s->len.mark_written();
  s->ub = n_ub;
  return MZGPU_OK;
}

static int32_t reduce_main(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                           bool minmax, u64 per_row);
static int32_t reduce_dev(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out) {
  MZ_TRY(reduce_begin(r));
  for (int j = 0; j < r->n_distinct; ++j)
    MZ_TRY(mzgpu_spine_set_physical_compaction(r->pairs[j], r->pairs[j]->upper));
  // explode_one: values move into the diff; the exploded rows become a stash segment
  // MIN / MAX / TopK keep the (key, value) rows themselves
  const bool minmax =
      r->agg_kind == MZGPU_AGG_MIN || r->agg_kind == MZGPU_AGG_MAX || r->agg_kind == MZGPU_AGG_TOPK;
  // output rows per distinct (key, time) of the new batch
  u64 per_row = 2;
  if (r->agg_kind == MZGPU_AGG_TOPK) {
    const u64 w = r->topk.limit >= 0 && r->topk.limit < 32 ? (u64)r->topk.limit : 32;
    per_row = 2 * w + 2;
  }
  // Distinct lanes first.  Their pair batches join the pair arrangements at the end whatever happens in
  // between, and a failure once a pair batcher may have been sealed kills the operator, as one after the
  // main seal does.
  mzgpu_batch* pair_new[MZGPU_MAX_ACCUM_LANES] = {};
  bool pairs_sealed = false;
  auto finish_pairs = [&](int32_t st) -> int32_t {
    for (int j = 0; j < r->n_distinct; ++j) {
      if (pair_new[j] == nullptr) continue;
      const int32_t ins = trace_join(r->pairs[j], pair_new[j]);
      pair_new[j] = nullptr;
      if (st == MZGPU_OK) st = ins;
    }
    return pairs_sealed ? reduce_kill_on_failure(r, st) : st;
  };
  if (r->n_distinct) {
    const int32_t ds = distinct_step(r, d_rows, n, n_ub, upper, pair_new, &pairs_sealed);
    if (ds != MZGPU_OK) return finish_pairs(ds);
  }
  return finish_pairs(reduce_main(r, d_rows, n, n_ub, upper, out, minmax, per_row));
}

// explode -> arrange -> reduce_abelian of one activation (after the distinct lanes' part)
static int32_t reduce_main(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                           bool minmax, u64 per_row) {
  mzgpu_ctx* ctx = r->ctx;
  const bool lanes = r->shape == ReduceShape::LANES;
  // a lanes operator whose lanes are all distinct has no plain explode
  const bool plain = !lanes || r->lanes.distinct_mask != (1u << r->lanes.n) - 1;
  if (n_ub && plain) {
    Seg s;
    if (minmax) {
      MZ_TRY(s.rows.alloc(ctx, n_ub * 32));
      MZ_CUDA(ctx, cudaMemcpyAsync(s.rows.p, d_rows, n_ub * 32, cudaMemcpyDeviceToDevice, ctx->stream));
    } else {
      MZ_TRY(s.rows.alloc(ctx, n_ub * (lanes ? mz_lane_arr_bytes(r->cls) : 80)));
      if (lanes)
        MZ_TRY(mz_explode_lanes(ctx, r->cls, d_rows, n, n_ub, r->lanes, s.rows.as<u64>()));
      else
        MZ_TRY(mz_explode(ctx, d_rows, n, n_ub, r->agg_kind, s.rows.as<u64>()));
    }
    MZ_TRY(seg_len_of_input(ctx, n, n_ub, &s));
    MZ_TRY(batcher_push_seg(r->batcher, std::move(s)));
  }
  // arrange: seal the accumulable arrangement's batch at the new frontier
  mzgpu_batch* batch = nullptr;
  MZ_TRY(batcher_seal(r->batcher, upper, &batch, nullptr));
  // reduce_abelian over the keys of the new batch
  TraceView tv;
  int32_t st = trace_view_of(r->input, &tv);
  const u64 b_ub = batch->len_ub;
  const int lc = lanes ? r->cls : 1;
  const u64 out_rb = (u64)mz_lane_out_bytes(lc);
  const LaneSet* ls = lanes ? &r->lanes : nullptr;
  const mzgpu_having* hv = r->has_having ? &r->having : nullptr;
  // The single-pass bound is checked against the batch's length bound; when that is loose (a
  // device-resident input buffer's capacity), the length is read back and checked again before the
  // two-pass form is used.
  u64 s_ub = b_ub;
  if (st == MZGPU_OK && b_ub > 0 && !single_pass_fits(b_ub, per_row)) {
    st = batch_resolve(batch);
    if (st == MZGPU_OK) s_ub = batch->st.v[0];
  }
  if (st == MZGPU_OK && s_ub > 0) {
    if (single_pass_fits(s_ub, per_row)) {
      DevMem corr;
      Lazy4 clen;
      st = corr.alloc(ctx, per_row * s_ub * out_rb);
      if (st == MZGPU_OK) st = clen.make_pending(ctx);
      if (st == MZGPU_OK) {
        if (minmax)
          st = mz_reduce_minmax_async(ctx, batch->rows.as<u64>(), batch_dlen(batch), s_ub, tv, r->agg_kind,
                                      r->topk, corr.as<u64>(), per_row * s_ub, clen.dptr());
        else
          st = mz_reduce_corrections_async(ctx, lc, batch->rows.as<u64>(), batch_dlen(batch), s_ub, tv,
                                           r->agg_kind, ls, corr.as<u64>(), per_row * s_ub, clen.dptr(), hv);
        clen.mark_written();
      }
      if (st == MZGPU_OK && !minmax) {
        // the accumulable kinds' corrections leave the kernel consolidated (reduce.cu:
        // sort_key_corrections): keys ascending, each key's few rows sorted by its thread
        st = buf_append_dev(out, corr.p, dlen_of(clen, 0), per_row * s_ub);
      } else if (st == MZGPU_OK) {
        st = append_consolidated(ctx, 64, corr.p, dlen_of(clen, 0), per_row * s_ub, out);
      }
    } else {
      DevMem corr;
      u64 n_corr = 0;
      if (minmax) {
        MZ_SET_ERR(ctx, "MIN/MAX/TopK reduce: batch of %llu rows exceeds the single-pass bound",
                   (unsigned long long)s_ub);
        st = MZGPU_E_UNSUPPORTED;
      }
      if (st == MZGPU_OK)
        st = mz_reduce_corrections(ctx, lc, batch->rows.as<u64>(), batch->st.v[0], tv, r->agg_kind, ls, &corr,
                                   &n_corr, hv);
      if (st == MZGPU_OK && n_corr && lc > 1) {
        // consolidated by construction, as in the single-pass form (and no RowT for these widths)
        st = buf_append_dev(out, corr.p, dlen_imm(n_corr), n_corr);
      } else if (st == MZGPU_OK) {
        st = append_consolidated(ctx, 64, corr.p, dlen_imm(n_corr), n_corr, out);
      }
    }
  }
  return reduce_seal_tail(r, batch, st);
}

// ------------------------------------------------------- reduce over several value columns
extern "C" int32_t mzgpu_reduce_lanes_row_bytes(uint32_t n_lanes, uint32_t* arr_row_bytes, uint32_t* out_row_bytes) {
  if (n_lanes == 0 || n_lanes > MZGPU_MAX_ACCUM_LANES) return MZGPU_E_INVALID;
  const int c = mz_lane_class(n_lanes);
  if (arr_row_bytes != nullptr) *arr_row_bytes = (uint32_t)mz_lane_arr_bytes(c);
  if (out_row_bytes != nullptr) *out_row_bytes = (uint32_t)mz_lane_out_bytes(c);
  return MZGPU_OK;
}

// The checks every lane constructor starts with: an output pointer, the lanes (n of them) and R32 / R40 input.
static int32_t lane_args_check(mzgpu_ctx* ctx, const char* name, uint32_t in_row_bytes, const void* lanes, uint32_t n,
                               mzgpu_reduce** out) {
  if (out == nullptr || (lanes == nullptr && n) || (in_row_bytes != 32 && in_row_bytes != 40)) {
    MZ_SET_ERR(ctx, "%s: bad arguments (input rows of %u bytes)", name, in_row_bytes);
    return MZGPU_E_INVALID;
  }
  return MZGPU_OK;
}
// Why a lane's field is not a bit-field of a value word of the input rows, or null when it is.
static const char* value_field_bad(const mzgpu_field& f, uint32_t in_row_bytes) {
  if (f.src != MZGPU_SRC_VAL1 && !(f.src == MZGPU_SRC_VAL2 && in_row_bytes == 40))
    return "source word is not a value word of the input row";
  if (f.bits == 0 || f.bits > 64 || f.shift > 63 || (u32)f.shift + f.bits > 64) return "field is empty or out of range";
  return nullptr;
}

extern "C" int32_t mzgpu_reduce_lanes_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                                          uint32_t n_lanes, mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  MZ_TRY(lane_args_check(ctx, "reduce_lanes", in_row_bytes, lanes, n_lanes, out));
  if (n_lanes == 0 || n_lanes > MZGPU_MAX_ACCUM_LANES) {
    MZ_SET_ERR(ctx, "reduce_lanes: %u lanes (1..%d)", n_lanes, MZGPU_MAX_ACCUM_LANES);
    return MZGPU_E_INVALID;
  }
  LaneSet ls = {};
  for (uint32_t l = 0; l < n_lanes; ++l) {
    const mzgpu_accum_lane& L = lanes[l];
    const mzgpu_field& f = L.field;
    const int32_t base = L.kind & ~MZGPU_ACCUM_DISTINCT;
    const bool distinct = (L.kind & MZGPU_ACCUM_DISTINCT) != 0;
    const bool f64 = base == MZGPU_AGG_COUNT_SUM_F64;
    const char* bad = value_field_bad(f, in_row_bytes);
    if (base != MZGPU_AGG_COUNT_SUM_I64 && !f64)
      bad = "kind is not COUNT_SUM_I64 / COUNT_SUM_F64, optionally | MZGPU_ACCUM_DISTINCT";
    else if (bad == nullptr && f64 && (f.shift != 0 || f.bits != 64))
      bad = "a float64 lane must pick a whole word";
    if (bad != nullptr) {
      MZ_SET_ERR(ctx, "reduce_lanes: lane %u: %s", l, bad);
      return MZGPU_E_INVALID;
    }
    if (distinct && f64) {
      MZ_SET_ERR(ctx, "reduce_lanes: lane %u: DISTINCT over float64 is not supported (which floats the "
                      "reference's Row arrangement treats as one value is not pinned)", l);
      return MZGPU_E_UNSUPPORTED;
    }
    ls.lane[l] = L;
    if (f64) ls.f64_mask |= 1u << l;
    if (distinct) ls.distinct_mask |= 1u << l;
  }
  ls.n = n_lanes;
  ls.in_words = in_row_bytes / 8;
  const int c = mz_lane_class(n_lanes);
  std::unique_ptr<mzgpu_reduce> r;
  MZ_TRY(reduce_alloc(ctx, ReduceShape::LANES, (uint32_t)mz_lane_arr_bytes(c), &r));
  r->cls = c;
  r->lanes = ls;
  r->agg_kind = (ls.f64_mask & 1u) ? MZGPU_AGG_COUNT_SUM_F64 : MZGPU_AGG_COUNT_SUM_I64;
  for (uint32_t l = 0; l < n_lanes; ++l) {
    if (((ls.distinct_mask >> l) & 1u) == 0) continue;
    const int j = r->n_distinct++;
    r->distinct_lane[j] = l;
    MZ_TRY(mzgpu_batcher_new(ctx, 32, &r->pair_batcher[j]));
    MZ_TRY(mzgpu_spine_new(ctx, 32, 1, &r->pairs[j]));
  }
  *out = r.release();
  return MZGPU_OK;
}

// The HAVING program's checks (include/mzgpu.h): a type per stack slot, simulated op by op.
// MZGPU_E_INVALID for a malformed program, MZGPU_E_UNSUPPORTED for a well-formed one outside the subset.
static int32_t validate_having(mzgpu_ctx* ctx, const mzgpu_having& h, const LaneSet& ls) {
  enum Ty { INT32, INT64, NUM, FLOAT, BOOL };
  auto bad = [&](int32_t st, uint32_t p, uint32_t i, const char* why) {
    MZ_SET_ERR(ctx, "reduce_lanes having: predicate %u, op %u: %s", p, i, why);
    return st;
  };
  if (h.n_predicates > MZGPU_HAVING_MAX_PREDICATES || h.n_consts > MZGPU_HAVING_MAX_CONSTS) {
    MZ_SET_ERR(ctx, "reduce_lanes having: %u predicates (0..%d), %u constants (0..%d)", h.n_predicates,
               MZGPU_HAVING_MAX_PREDICATES, h.n_consts, MZGPU_HAVING_MAX_CONSTS);
    return MZGPU_E_INVALID;
  }
  int32_t unsupported = MZGPU_OK;  // reported once the whole program is known to be well-formed
  const char* unsupported_why = nullptr;
  uint32_t up = 0, ui = 0;
  auto outside = [&](uint32_t p, uint32_t i, const char* why) {
    if (unsupported == MZGPU_OK) {
      unsupported = MZGPU_E_UNSUPPORTED;
      unsupported_why = why;
      up = p;
      ui = i;
    }
  };
  for (uint32_t p = 0; p < h.n_predicates; ++p) {
    const uint32_t n_ops = h.n_ops[p];
    if (n_ops == 0 || n_ops > MZGPU_HAVING_MAX_OPS) return bad(MZGPU_E_INVALID, p, 0, "op count (1..16)");
    Ty ty[MZGPU_HAVING_MAX_STACK];
    int sp = 0;
    for (uint32_t i = 0; i < n_ops; ++i) {
      const mzgpu_having_op& o = h.ops[p][i];
      const uint32_t code = o.code;
      if (code >= MZGPU_HOP_KEY && code <= MZGPU_HOP_FLOAT) {
        if (sp == MZGPU_HAVING_MAX_STACK) return bad(MZGPU_E_INVALID, p, i, "stack overflow (depth 8)");
        Ty t;
        if (code == MZGPU_HOP_KEY) {
          if (o.bits == 0 || o.bits > 64 || (uint32_t)o.shift + o.bits > 64 || o.sign_extend > 1)
            return bad(MZGPU_E_INVALID, p, i, "key field is empty or out of range");
          t = (o.bits < 32 || (o.bits == 32 && o.sign_extend)) ? INT32 : INT64;
        } else if (code == MZGPU_HOP_COUNT || code == MZGPU_HOP_SUM) {
          if (o.arg >= ls.n) return bad(MZGPU_E_INVALID, p, i, "lane out of range");
          t = code == MZGPU_HOP_COUNT ? INT64 : (((ls.f64_mask >> o.arg) & 1u) ? FLOAT : NUM);
        } else {
          if (o.konst >= h.n_consts) return bad(MZGPU_E_INVALID, p, i, "constant index out of range");
          const mzgpu_having_const& k = h.consts[o.konst];
          const bool fits64 = k.hi == ((int64_t)k.lo < 0 ? ~0ull : 0ull);
          if (code == MZGPU_HOP_INT) {
            if (!fits64) return bad(MZGPU_E_INVALID, p, i, "INT constant outside i64");
            const int64_t v = (int64_t)k.lo;
            t = v >= INT32_MIN && v <= INT32_MAX ? INT32 : INT64;
          } else if (code == MZGPU_HOP_FLOAT) {
            if (k.hi != 0) return bad(MZGPU_E_INVALID, p, i, "FLOAT constant with a non-zero high word");
            t = FLOAT;
          } else {
            t = NUM;
          }
        }
        ty[sp++] = t;
        continue;
      }
      if (code == MZGPU_HOP_NOT) {
        if (sp < 1) return bad(MZGPU_E_INVALID, p, i, "stack underflow");
        if (ty[sp - 1] != BOOL) return bad(MZGPU_E_INVALID, p, i, "NOT of a non-BOOL");
        continue;
      }
      if (code < MZGPU_HOP_ADD || code > MZGPU_HOP_OR) return bad(MZGPU_E_INVALID, p, i, "unknown opcode");
      if (sp < 2) return bad(MZGPU_E_INVALID, p, i, "stack underflow");
      const Ty a = ty[sp - 2], b = ty[sp - 1];
      --sp;
      const bool ia = a == INT32 || a == INT64, ib = b == INT32 || b == INT64;
      if (code == MZGPU_HOP_AND || code == MZGPU_HOP_OR) {
        if (a != BOOL || b != BOOL) return bad(MZGPU_E_INVALID, p, i, "AND / OR of a non-BOOL");
      } else if (code == MZGPU_HOP_CMP) {
        if (o.arg > MZGPU_CMP_GE) return bad(MZGPU_E_INVALID, p, i, "unknown compare op");
        if ((a == BOOL) != (b == BOOL)) return bad(MZGPU_E_INVALID, p, i, "BOOL compared with a value");
        if (a == BOOL) outside(p, i, "BOOL comparisons");
        else if ((a == FLOAT) != (b == FLOAT)) outside(p, i, "FLOAT compared with INT / NUM");
        ty[sp - 1] = BOOL;
      } else {
        if (o.arg != 32 && o.arg != 64) return bad(MZGPU_E_INVALID, p, i, "width is not 32 or 64");
        if (a == BOOL || b == BOOL) return bad(MZGPU_E_INVALID, p, i, "arithmetic on a BOOL");
        if (!ia || !ib) {
          outside(p, i, "arithmetic on a NUM or FLOAT");
          ty[sp - 1] = a;
        } else if (o.arg == 32 && (a != INT32 || b != INT32)) {
          return bad(MZGPU_E_INVALID, p, i, "32-bit operation on an operand that is not int32");
        } else {
          ty[sp - 1] = o.arg == 32 ? INT32 : INT64;
        }
      }
    }
    if (sp != 1 || ty[0] != BOOL) return bad(MZGPU_E_INVALID, p, n_ops, "the predicate does not leave one BOOL");
  }
  if (unsupported != MZGPU_OK) return bad(unsupported, up, ui, unsupported_why);
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_reduce_lanes_new_having(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                                                 uint32_t n_lanes, const mzgpu_having* having, mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  mzgpu_reduce* r = nullptr;
  MZ_TRY(mzgpu_reduce_lanes_new(ctx, in_row_bytes, lanes, n_lanes, &r));
  if (having != nullptr && having->n_predicates != 0) {
    const int32_t st = validate_having(ctx, *having, r->lanes);
    if (st != MZGPU_OK) {
      mzgpu_reduce_free(r);
      return st;
    }
    r->has_having = true;
    r->having = *having;
  }
  *out = r;
  return MZGPU_OK;
}

extern "C" mzgpu_spine* mzgpu_reduce_lanes_distinct_trace(mzgpu_reduce* r, uint32_t lane) {
  if (r == nullptr) return nullptr;
  for (int j = 0; j < r->n_distinct; ++j)
    if (r->distinct_lane[j] == lane) return r->pairs[j];
  return nullptr;
}

// ------------------------------------------------------- monotonic MIN / MAX reduce
extern "C" int32_t mzgpu_reduce_monotonic_row_bytes(uint32_t n_lanes, uint32_t* arr_row_bytes,
                                                    uint32_t* out_row_bytes) {
  if (n_lanes == 0 || n_lanes > MZGPU_MAX_ACCUM_LANES) return MZGPU_E_INVALID;
  const int c = mz_mono_class(n_lanes);
  if (arr_row_bytes != nullptr) *arr_row_bytes = (uint32_t)mz_mono_arr_bytes(c);
  if (out_row_bytes != nullptr) *out_row_bytes = (uint32_t)mz_mono_out_bytes(c);
  return MZGPU_OK;
}

// The MIN / MAX lanes of the monotonic and hierarchical reduces, checked on the host (`what` names the operator
// in the messages): MZGPU_E_INVALID for a malformed descriptor, then MZGPU_E_UNSUPPORTED for a float64 lane.
// Fills the lanes, their encodings (value ^ xm: every lane an unsigned max) and the value bits they read.
static int32_t minmax_lanes(mzgpu_ctx* ctx, const char* what, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                            uint32_t n_lanes, mzgpu_reduce** out, LaneSet* ls_out, MonoXor* mx_out, u64* mask) {
  MZ_TRY(lane_args_check(ctx, what, in_row_bytes, lanes, n_lanes, out));
  if (n_lanes == 0 || n_lanes > MZGPU_MAX_ACCUM_LANES) {
    MZ_SET_ERR(ctx, "%s: %u lanes (1..%d)", what, n_lanes, MZGPU_MAX_ACCUM_LANES);
    return MZGPU_E_INVALID;
  }
  LaneSet ls = {};
  MonoXor mx = {};
  mask[0] = mask[1] = 0;
  int unsupported = -1;  // the first float64 lane, reported once every lane is known to be well-formed
  for (uint32_t l = 0; l < n_lanes; ++l) {
    const mzgpu_accum_lane& L = lanes[l];
    const mzgpu_field& f = L.field;
    const int32_t base = L.kind & ~MZGPU_MONO_F64;
    const char* bad = value_field_bad(f, in_row_bytes);
    if (base != MZGPU_AGG_MIN && base != MZGPU_AGG_MAX)
      bad = "kind is not MZGPU_AGG_MIN / MZGPU_AGG_MAX, optionally | MZGPU_MONO_F64";
    if (bad != nullptr) {
      MZ_SET_ERR(ctx, "%s: lane %u: %s", what, l, bad);
      return MZGPU_E_INVALID;
    }
    if ((L.kind & MZGPU_MONO_F64) != 0 && unsupported < 0) unsupported = (int)l;
    ls.lane[l] = L;
    mx.xm[l] = (L.sign_extend ? 1ull << 63 : 0) ^ (base == MZGPU_AGG_MIN ? ~0ull : 0);
    mask[f.src == MZGPU_SRC_VAL2 ? 1 : 0] |= (f.bits == 64 ? ~0ull : ((1ull << f.bits) - 1)) << f.shift;
  }
  if (unsupported >= 0) {
    MZ_SET_ERR(ctx, "%s: lane %d: float64 MIN / MAX is not supported (OrderedFloat ties -0.0 with "
                    "+0.0 and NaN payloads, so the surviving bits would depend on arrival order)", what, unsupported);
    return MZGPU_E_UNSUPPORTED;
  }
  ls.n = n_lanes;
  ls.in_words = in_row_bytes / 8;
  mx.n = n_lanes;
  *ls_out = ls;
  *mx_out = mx;
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_reduce_monotonic_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                                              uint32_t n_lanes, int32_t must_consolidate, mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  LaneSet ls;
  MonoXor mx;
  u64 mask[2];
  MZ_TRY(minmax_lanes(ctx, "reduce_monotonic", in_row_bytes, lanes, n_lanes, out, &ls, &mx, mask));
  const int c = mz_mono_class(n_lanes);
  std::unique_ptr<mzgpu_reduce> r;
  MZ_TRY(reduce_alloc(ctx, ReduceShape::MONOTONIC, (uint32_t)mz_mono_arr_bytes(c), &r));
  r->cls = c;
  r->lanes = ls;
  r->mono = mx;
  r->must_consolidate = must_consolidate != 0;
  r->mono_mask[0] = mask[0];
  r->mono_mask[1] = mask[1];
  *out = r.release();
  return MZGPU_OK;
}

// One activation of build_monotonic: [consolidate ->] ensure_monotonic + explode -> arrange -> corrections.
static int32_t monotonic_dev(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                             mzgpu_buf* errs) {
  mzgpu_ctx* ctx = r->ctx;
  MZ_TRY(reduce_begin(r));
  const int c = r->cls;
  if (n_ub) {
    const u32 iw = r->lanes.in_words;
    DevMem masked, cons;
    Lazy4 clen;
    if (r->must_consolidate) {
      // consolidate_named_if: rows that agree on (key, lane values, time) fold, a +1 / -1 pair vanishes
      u64 ccap = 0;
      MZ_TRY(masked.alloc(ctx, n_ub * iw * 8));
      MZ_TRY(mz_monotonic_mask(ctx, d_rows, n, n_ub, iw, r->mono_mask[0], r->mono_mask[1], masked.as<u64>()));
      MZ_TRY(consolidate_dev(ctx, (int)iw * 8, masked.p, n, n_ub, &cons, &ccap, &clen));
      d_rows = cons.as<u64>();
      n = dlen_of(clen, 0);
      if (clen.known) n_ub = clen.v[0];
    }
    Seg s;
    DevMem erows;
    MZ_TRY(s.rows.alloc(ctx, n_ub * mz_mono_arr_bytes(c)));
    MZ_TRY(erows.alloc(ctx, n_ub * 16));
    MZ_TRY(s.len.make_pending(ctx));
    MZ_TRY(mz_monotonic_explode(ctx, c, d_rows, n, n_ub, r->lanes, r->mono, s.rows.as<u64>(), erows.as<u64>(),
                                s.len.dptr()));
    s.len.mark_written();
    s.ub = n_ub;
    // the rejected rows' error collection: (time, number of rejected rows)
    MZ_TRY(append_consolidated(ctx, 16, erows.p, dlen_of(s.len, 1), n_ub, errs));
    MZ_TRY(batcher_push_seg(r->batcher, std::move(s)));
  }
  mzgpu_batch* batch = nullptr;
  MZ_TRY(batcher_seal(r->batcher, upper, &batch, nullptr));
  TraceView tv;
  int32_t st = trace_view_of(r->input, &tv);
  const u64 b_ub = batch->len_ub;
  const u64 out_rb = (u64)mz_mono_out_bytes(c);
  if (st == MZGPU_OK && b_ub > 0) {
    if (single_pass_fits(b_ub, 2)) {  // (the bound alone: a loose one takes the two-pass form)
      DevMem corr;
      Lazy4 clen;
      st = corr.alloc(ctx, 2 * b_ub * out_rb);
      if (st == MZGPU_OK) st = clen.make_pending(ctx);
      if (st == MZGPU_OK) {
        st = mz_monotonic_corrections_async(ctx, c, batch->rows.as<u64>(), batch_dlen(batch), b_ub, tv, r->mono,
                                            corr.as<u64>(), 2 * b_ub, clen.dptr());
        clen.mark_written();
      }
      // consolidated by construction: keys ascending, each key's rows sorted by its thread
      if (st == MZGPU_OK) st = buf_append_dev(out, corr.p, dlen_of(clen, 0), 2 * b_ub);
    } else {
      DevMem corr;
      u64 n_corr = 0;
      st = batch_resolve(batch);
      if (st == MZGPU_OK)
        st = mz_monotonic_corrections(ctx, c, batch->rows.as<u64>(), batch->st.v[0], tv, r->mono, &corr, &n_corr);
      if (st == MZGPU_OK && n_corr) st = buf_append_dev(out, corr.p, dlen_imm(n_corr), n_corr);
    }
  }
  return reduce_seal_tail(r, batch, st);
}

// ------------------------------------------------------- hierarchical MIN / MAX reduce
extern "C" int32_t mzgpu_reduce_hierarchical_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                                                 uint32_t n_lanes, mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  LaneSet ls;
  MonoXor mx;
  u64 mask[2];
  MZ_TRY(minmax_lanes(ctx, "reduce_hierarchical", in_row_bytes, lanes, n_lanes, out, &ls, &mx, mask));
  std::unique_ptr<mzgpu_reduce> r;
  // the arrangement holds the masked input rows themselves, with ordinary SUM diffs
  MZ_TRY(reduce_alloc(ctx, ReduceShape::HIERARCHICAL, in_row_bytes, &r));
  r->cls = mz_mono_class(n_lanes);
  r->lanes = ls;
  r->mono = mx;
  r->mono_mask[0] = mask[0];
  r->mono_mask[1] = mask[1];
  *out = r.release();
  return MZGPU_OK;
}

// One activation of build_bucketed: mask -> arrange -> per-key MIN / MAX of the live rows, and the keys'
// non-positive-accumulation errors.
static int32_t hierarchical_dev(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                                mzgpu_buf* errs) {
  mzgpu_ctx* ctx = r->ctx;
  MZ_TRY(reduce_begin(r));
  const int c = r->cls;
  const u32 iw = r->lanes.in_words;
  if (n_ub) {
    // (key, the bits the lanes read, time, diff): rows that differ only in unread bits are one value row
    Seg s;
    MZ_TRY(s.rows.alloc(ctx, n_ub * iw * 8));
    MZ_TRY(mz_monotonic_mask(ctx, d_rows, n, n_ub, iw, r->mono_mask[0], r->mono_mask[1], s.rows.as<u64>()));
    MZ_TRY(seg_len_of_input(ctx, n, n_ub, &s));
    MZ_TRY(batcher_push_seg(r->batcher, std::move(s)));
  }
  mzgpu_batch* batch = nullptr;
  MZ_TRY(batcher_seal(r->batcher, upper, &batch, nullptr));
  TraceView tv;
  int32_t st = trace_view_of(r->input, &tv);
  const u64 b_ub = batch->len_ub;
  if (st == MZGPU_OK && b_ub > 0) {
    DevMem corr, erows;
    Lazy4 elen;
    u64 e_ub = b_ub;
    st = elen.make_pending(ctx);
    if (single_pass_fits(b_ub, 2)) {  // (the bound alone: a loose one takes the two-pass form)
      Lazy4 clen;
      if (st == MZGPU_OK) st = corr.alloc(ctx, 2 * b_ub * mz_mono_out_bytes(c));
      if (st == MZGPU_OK) st = erows.alloc(ctx, b_ub * 32);
      if (st == MZGPU_OK) st = clen.make_pending(ctx);
      if (st == MZGPU_OK) {
        st = mz_hier_corrections_async(ctx, c, batch->rows.as<u64>(), batch_dlen(batch), b_ub, tv, r->lanes, r->mono,
                                       corr.as<u64>(), 2 * b_ub, clen.dptr(), erows.as<u64>(), b_ub, elen.dptr());
        clen.mark_written();
        elen.mark_written();
      }
      // consolidated by construction: keys ascending, each key's rows sorted by its thread
      if (st == MZGPU_OK) st = buf_append_dev(out, corr.p, dlen_of(clen, 0), 2 * b_ub);
    } else {
      u64 n_corr = 0;
      if (st == MZGPU_OK) st = batch_resolve(batch);
      if (st == MZGPU_OK) e_ub = batch->st.v[0];
      if (st == MZGPU_OK) st = erows.alloc(ctx, std::max<u64>(e_ub, 1) * 32);
      if (st == MZGPU_OK) {
        st = mz_hier_corrections(ctx, c, batch->rows.as<u64>(), e_ub, tv, r->lanes, r->mono, &corr, &n_corr,
                                 erows.as<u64>(), e_ub, elen.dptr());
        elen.mark_written();
      }
      if (st == MZGPU_OK && n_corr) st = buf_append_dev(out, corr.p, dlen_imm(n_corr), n_corr);
    }
    // the error rows leave the kernel unordered: (key, 0, time, +-1), at most one per key and time
    if (st == MZGPU_OK) st = append_consolidated(ctx, 32, erows.p, dlen_of(elen, 0), e_ub, errs);
  }
  return reduce_seal_tail(r, batch, st);
}

// ------------------------------------------------------- monotonic TopK
// The order lanes of a TopK operator, checked as the header states (MZGPU_E_INVALID for a malformed
// descriptor, then MZGPU_E_UNSUPPORTED for a float64 lane or a negative limit) into *to.
static int32_t topk_order(mzgpu_ctx* ctx, const char* name, uint32_t in_row_bytes, const mzgpu_order_lane* order,
                          uint32_t n_order, int64_t limit, mzgpu_reduce** out, TopKOrder* to_out) {
  MZ_TRY(lane_args_check(ctx, name, in_row_bytes, order, n_order, out));
  if (n_order > MZGPU_MAX_ORDER_LANES) {
    MZ_SET_ERR(ctx, "%s: %u order lanes (0..%d)", name, n_order, MZGPU_MAX_ORDER_LANES);
    return MZGPU_E_INVALID;
  }
  TopKOrder to = {};
  int unsupported = -1;  // the first float64 lane, reported once every lane is known to be well-formed
  for (uint32_t j = 0; j < n_order; ++j) {
    const mzgpu_order_lane& L = order[j];
    const mzgpu_field& f = L.field;
    const char* bad = value_field_bad(f, in_row_bytes);
    if ((L.flags & ~(uint32_t)MZGPU_ORDER_F64) != 0) bad = "unknown flag bits";
    if (bad != nullptr) {
      MZ_SET_ERR(ctx, "%s: order lane %u: %s", name, j, bad);
      return MZGPU_E_INVALID;
    }
    if ((L.flags & MZGPU_ORDER_F64) != 0 && unsupported < 0) unsupported = (int)j;
    to.f[j] = f;
    to.sign_extend[j] = L.sign_extend != 0;
    to.xm[j] = (L.sign_extend ? 1ull << 63 : 0) ^ (L.descending ? ~0ull : 0);
  }
  if (unsupported >= 0) {
    MZ_SET_ERR(ctx, "%s: order lane %d: float64 order columns are not supported (OrderedFloat ties "
                    "-0.0 with +0.0 and NaN payloads)", name, unsupported);
    return MZGPU_E_UNSUPPORTED;
  }
  if (limit < 0) {
    MZ_SET_ERR(ctx, "%s: negative limit %lld", name, (long long)limit);
    return MZGPU_E_UNSUPPORTED;
  }
  to.n = n_order;
  to.in_words = in_row_bytes / 8;
  to.limit = limit;
  *to_out = to;
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_topk_monotonic_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_order_lane* order,
                                            uint32_t n_order, int64_t limit, int32_t must_consolidate,
                                            mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  TopKOrder to;
  MZ_TRY(topk_order(ctx, "topk_monotonic", in_row_bytes, order, n_order, limit, out, &to));
  std::unique_ptr<mzgpu_reduce> r;
  MZ_TRY(reduce_alloc(ctx, ReduceShape::TOPK_MONOTONIC, MZGPU_ROW_RTOPK, &r));
  r->tko = to;
  r->must_consolidate = must_consolidate != 0;
  *out = r.release();
  return MZGPU_OK;
}

// One activation: [consolidate ->] ensure_monotonic + explode -> sort -> window changes -> seal the changes.
static int32_t topk_monotonic_dev(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                                  mzgpu_buf* errs) {
  mzgpu_ctx* ctx = r->ctx;
  MZ_TRY(reduce_begin(r));
  const TopKOrder& to = r->tko;
  const u32 iw = to.in_words;
  const u64 RB = MZGPU_ROW_RTOPK;
  int32_t st = MZGPU_OK;
  if (n_ub) {
    DevMem cons;
    Lazy4 clen;
    if (r->must_consolidate) {  // consolidate_named_if on (group_key, row): whole rows, then time
      u64 ccap = 0;
      MZ_TRY(consolidate_dev(ctx, (int)iw * 8, d_rows, n, n_ub, &cons, &ccap, &clen));
      d_rows = cons.as<u64>();
      n = dlen_of(clen, 0);
      if (clen.known) n_ub = clen.v[0];
    }
    DevMem arr, erows, sorted;
    Lazy4 alen, slen;
    u64 scap = 0;
    MZ_TRY(arr.alloc(ctx, n_ub * RB));
    MZ_TRY(erows.alloc(ctx, n_ub * 16));
    MZ_TRY(alen.make_pending(ctx));
    MZ_TRY(mz_topk_explode(ctx, d_rows, n, n_ub, to, arr.as<u64>(), erows.as<u64>(), alen.dptr()));
    alen.mark_written();
    // the rejected rows' error collection: (time, number of rejected rows)
    MZ_TRY(append_consolidated(ctx, 16, erows.p, dlen_of(alen, 1), n_ub, errs));
    // the kept rows sorted and consolidated by (key, order, row, time); never arranged themselves
    MZ_TRY(consolidate_dev(ctx, (int)RB, arr.p, dlen_of(alen, 0), n_ub, &sorted, &scap, &slen));
    arr.release();
    const u64 s_ub = slen.known ? slen.v[0] : n_ub;
    TraceView tv;
    MZ_TRY(trace_view_of(r->input, &tv));
    // Output bound of one new row of multiplicity m: it enters at most once, and the units it adds evict or
    // cut at most min(m, limit) rows, so 1 + limit rows per new row (exactly one without a limit).
    const i64 L = to.limit;
    const u64 per_row = L == INT64_MAX ? 1 : (u64)L + 1;
    Seg w;
    w.ub = 0;
    if (L != 0 && s_ub > 0) {
      if ((u64)L < MZ_BOUND_MAX_ROWS && single_pass_fits(s_ub, per_row)) {
        const u64 cap = per_row * s_ub;
        DevMem proj;
        st = w.rows.alloc(ctx, cap * RB);
        if (st == MZGPU_OK) st = proj.alloc(ctx, cap * iw * 8);
        if (st == MZGPU_OK) st = w.len.make_pending(ctx);
        if (st == MZGPU_OK) {
          st = mz_topk_window_async(ctx, sorted.as<u64>(), dlen_of(slen, 0), s_ub, tv, to, w.rows.as<u64>(),
                                    proj.as<u64>(), cap, w.len.dptr());
          w.len.mark_written();
          w.ub = cap;
        }
        // consolidated by construction: keys ascending, each key's rows sorted by its thread
        if (st == MZGPU_OK) st = buf_append_dev(out, proj.p, dlen_of(w.len, 0), cap);
      } else {
        DevMem proj;
        u64 n_win = 0;
        if (st == MZGPU_OK) st = slen.resolve();
        if (st == MZGPU_OK)
          st = mz_topk_window(ctx, sorted.as<u64>(), slen.v[0], tv, to, &w.rows, &proj, &n_win);
        if (st == MZGPU_OK && n_win) {
          w.len.set(ctx, n_win);
          w.ub = n_win;
          st = buf_append_dev(out, proj.p, dlen_imm(n_win), n_win);
        }
      }
    }
    if (st != MZGPU_OK) return st;  // nothing sealed yet: the operator stays usable
    if (w.ub) MZ_TRY(batcher_push_seg(r->batcher, std::move(w)));
  }
  mzgpu_batch* batch = nullptr;
  MZ_TRY(batcher_seal(r->batcher, upper, &batch, nullptr));
  return reduce_seal_tail(r, batch, MZGPU_OK);
}

// ------------------------------------------------------- basic TopK
extern "C" int32_t mzgpu_topk_basic_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_order_lane* order,
                                        uint32_t n_order, int64_t limit, uint64_t offset, mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  TopKOrder to;
  MZ_TRY(topk_order(ctx, "topk_basic", in_row_bytes, order, n_order, limit, out, &to));
  if (limit != MZGPU_TOPK_NO_LIMIT && offset > (u64)(INT64_MAX - limit)) {
    MZ_SET_ERR(ctx, "topk_basic: offset %llu + limit %lld overflows a 64-bit count (a limit expression)",
               (unsigned long long)offset, (long long)limit);
    return MZGPU_E_UNSUPPORTED;
  }
  std::unique_ptr<mzgpu_reduce> r;
  MZ_TRY(reduce_alloc(ctx, ReduceShape::TOPK_BASIC, MZGPU_ROW_RTOPK, &r));
  r->tko = to;
  // (no count reaches 2^63: an offset past it leaves every window empty, as INT64_MAX does)
  r->topk_offset = (i64)std::min<u64>(offset, (u64)INT64_MAX);
  MZ_TRY(mzgpu_batcher_new(ctx, 32, &r->neg_batcher));
  MZ_TRY(mzgpu_spine_new(ctx, 32, 1, &r->negs));
  *out = r.release();
  return MZGPU_OK;
}
extern "C" mzgpu_spine* mzgpu_topk_basic_negatives_trace(mzgpu_reduce* r) { return r ? r->negs : nullptr; }

// One activation of build_topk_negated_stage: explode -> arrange (sort, consolidate, seal) -> per key the
// negative counts, error states and window changes of the new times -> seal the negatives.
static int32_t topk_basic_dev(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                              mzgpu_buf* errs) {
  mzgpu_ctx* ctx = r->ctx;
  MZ_TRY(reduce_begin(r));
  const TopKOrder& to = r->tko;
  const u32 iw = to.in_words;
  if (n_ub) {
    Seg s;
    MZ_TRY(s.rows.alloc(ctx, n_ub * MZGPU_ROW_RTOPK));
    MZ_TRY(mz_topk_basic_explode(ctx, d_rows, n, n_ub, to, s.rows.as<u64>()));
    MZ_TRY(seg_len_of_input(ctx, n, n_ub, &s));
    MZ_TRY(batcher_push_seg(r->batcher, std::move(s)));
  }
  mzgpu_batch* batch = nullptr;
  MZ_TRY(batcher_seal(r->batcher, upper, &batch, nullptr));
  TraceView tv, nv;
  int32_t st = trace_view_of(r->input, &tv);
  if (st == MZGPU_OK) st = trace_view_of(r->negs, &nv);
  const u64 b_ub = batch->len_ub;
  Seg ns;  // the negatives deltas: the negatives batcher's new rows
  if (st == MZGPU_OK && b_ub > 0) {
    DevMem corr, erows;
    Lazy4 slen;  // [0] error rows, [1] negatives rows
    u64 s_ub = b_ub;
    st = slen.make_pending(ctx);
    // Output rows per new row, finite limit: a change at one new time of a key is a row whose share of the
    // window differs between the previous and the current time, so it holds a unit of the old window or of the
    // new one; each window is at most `limit` units, hence at most 2 * limit rows per new time, and a key has
    // no more new times than new rows.
    const i64 L = to.limit;
    if (L != MZGPU_TOPK_NO_LIMIT && (u64)L < MZ_BOUND_MAX_ROWS && single_pass_fits(b_ub, 2 * (u64)L)) {
      const u64 cap = 2 * (u64)L * b_ub;
      Lazy4 clen;
      if (st == MZGPU_OK) st = corr.alloc(ctx, std::max<u64>(cap, 1) * iw * 8);
      if (st == MZGPU_OK) st = erows.alloc(ctx, b_ub * 32);
      if (st == MZGPU_OK) st = ns.rows.alloc(ctx, b_ub * 32);
      if (st == MZGPU_OK) st = clen.make_pending(ctx);
      if (st == MZGPU_OK) {
        st = mz_topk_basic_async(ctx, batch->rows.as<u64>(), batch_dlen(batch), b_ub, tv, nv, to, r->topk_offset,
                                 corr.as<u64>(), cap, clen.dptr(), erows.as<u64>(), ns.rows.as<u64>(), b_ub,
                                 slen.dptr());
        clen.mark_written();
        slen.mark_written();
      }
      // consolidated by construction: keys ascending, each key's rows sorted by its thread
      if (st == MZGPU_OK) st = buf_append_dev(out, corr.p, dlen_of(clen, 0), cap);
    } else {
      u64 n_corr = 0;
      if (st == MZGPU_OK) st = batch_resolve(batch);
      if (st == MZGPU_OK) s_ub = batch->st.v[0];
      if (st == MZGPU_OK) st = erows.alloc(ctx, std::max<u64>(s_ub, 1) * 32);
      if (st == MZGPU_OK) st = ns.rows.alloc(ctx, std::max<u64>(s_ub, 1) * 32);
      if (st == MZGPU_OK) {
        st = mz_topk_basic(ctx, batch->rows.as<u64>(), s_ub, tv, nv, to, r->topk_offset, &corr, &n_corr,
                           erows.as<u64>(), ns.rows.as<u64>(), s_ub, slen.dptr());
        slen.mark_written();
      }
      if (st == MZGPU_OK && n_corr) st = buf_append_dev(out, corr.p, dlen_imm(n_corr), n_corr);
    }
    // the error rows leave the kernel unordered: (key, 0, time, +-1), at most one per key and time
    if (st == MZGPU_OK) st = append_consolidated(ctx, 32, erows.p, dlen_of(slen, 0), s_ub, errs);
    // the negatives deltas, unordered too: the seal below sorts and consolidates them
    if (st == MZGPU_OK && s_ub > 0) {
      ns.len = std::move(slen);
      ns.word = 1;
      ns.ub = s_ub;
    }
  }
  int32_t nst = st;
  if (nst == MZGPU_OK && ns.ub) nst = batcher_push_seg(r->neg_batcher, std::move(ns));
  mzgpu_batch* nb = nullptr;
  if (nst == MZGPU_OK) nst = batcher_seal(r->neg_batcher, upper, &nb, nullptr);
  if (nb != nullptr) {
    const int32_t ins = trace_join(r->negs, nb);
    if (nst == MZGPU_OK) nst = ins;
  }
  if (nst == MZGPU_OK) nst = mzgpu_spine_set_logical_compaction(r->negs, upper);
  if (nst == MZGPU_OK) nst = mzgpu_spine_set_physical_compaction(r->negs, upper);
  return reduce_seal_tail(r, batch, nst);
}

// ------------------------------------------------------- step entry points
// The rows one step of an operator of `shape` takes: its name in messages, the input and output row bytes (r's
// own; meaningful when r has that shape) and the error row bytes (0: no error buffer).
struct ReduceIo {
  const char* name;
  uint32_t in_rb, out_rb, errs_rb;
};
static ReduceIo reduce_io(ReduceShape shape, const mzgpu_reduce* r) {
  const uint32_t lanes_in = r->lanes.in_words * 8, order_in = r->tko.in_words * 8;
  switch (shape) {
    case ReduceShape::ACCUM: return {"reduce_accumulable", 32, 64, 0};
    case ReduceShape::LANES: return {"reduce_lanes", lanes_in, (uint32_t)mz_lane_out_bytes(r->cls), 0};
    case ReduceShape::MONOTONIC: return {"reduce_monotonic", lanes_in, (uint32_t)mz_mono_out_bytes(r->cls), 16};
    case ReduceShape::HIERARCHICAL: return {"reduce_hierarchical", lanes_in, (uint32_t)mz_mono_out_bytes(r->cls), 32};
    case ReduceShape::TOPK_MONOTONIC: return {"topk_monotonic", order_in, order_in, 16};
    case ReduceShape::TOPK_BASIC: return {"topk_basic", order_in, order_in, 32};
  }
  return {};
}

// MZGPU_E_INVALID with the entry point's message unless r has `shape` and the input rows, out and errs (a second
// buffer) have its widths.  `rows` is the buffer form's input, null in the host form (rows of the operator's
// own width).
static int32_t reduce_io_check(const ReduceIo& io, ReduceShape shape, mzgpu_reduce* r, const mzgpu_buf* rows,
                               const mzgpu_buf* out, const mzgpu_buf* errs) {
  if (r->shape == shape && (rows == nullptr || rows->rb == io.in_rb) && out->rb == io.out_rb &&
      (io.errs_rb == 0 || (errs->rb == io.errs_rb && out != errs)))
    return MZGPU_OK;
  mzgpu_ctx* ctx = r->ctx;
  if (rows == nullptr && io.errs_rb)
    MZ_SET_ERR(ctx, "%s: output buffer of %u-byte rows / error buffer of %u-byte rows", io.name, out->rb, errs->rb);
  else if (rows == nullptr)
    MZ_SET_ERR(ctx, "%s: output buffer of %u-byte rows", io.name, out->rb);
  else if (io.errs_rb)
    MZ_SET_ERR(ctx, "%s: input rows of %u bytes / output rows of %u bytes / error rows of %u bytes", io.name,
               rows->rb, out->rb, errs->rb);
  else
    MZ_SET_ERR(ctx, "%s: input rows of %u bytes / output rows of %u bytes", io.name, rows->rb, out->rb);
  return MZGPU_E_INVALID;
}

// One activation of r over device rows, by its shape.
static int32_t reduce_step_dev(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                               mzgpu_buf* errs) {
  switch (r->shape) {
    case ReduceShape::ACCUM:
    case ReduceShape::LANES: return reduce_dev(r, d_rows, n, n_ub, upper, out);
    case ReduceShape::MONOTONIC: return monotonic_dev(r, d_rows, n, n_ub, upper, out, errs);
    case ReduceShape::HIERARCHICAL: return hierarchical_dev(r, d_rows, n, n_ub, upper, out, errs);
    case ReduceShape::TOPK_MONOTONIC: return topk_monotonic_dev(r, d_rows, n, n_ub, upper, out, errs);
    case ReduceShape::TOPK_BASIC: return topk_basic_dev(r, d_rows, n, n_ub, upper, out, errs);
  }
  return MZGPU_E_INVALID;
}

// The host form of a step: n rows of the operator's input width in `mem`.
static int32_t reduce_step(ReduceShape shape, mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem,
                           uint64_t upper, mzgpu_buf* out, mzgpu_buf* errs) {
  if (r == nullptr || out == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  const ReduceIo io = reduce_io(shape, r);
  if (io.errs_rb && errs == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(r->ctx);
  MZ_TRY(reduce_io_check(io, shape, r, nullptr, out, errs));
  DevMem in;
  const u64* d_rows;
  MZ_TRY(entry_rows_in(r->ctx, rows, n, mem, io.in_rb, &in, &d_rows));
  return reduce_step_dev(r, d_rows, dlen_imm(n), n, upper, out, errs);
}
// The buffer form of a step: the rows of a device buffer, read without waiting for its length.
static int32_t reduce_step_buf(ReduceShape shape, mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out,
                               mzgpu_buf* errs) {
  if (r == nullptr || rows == nullptr || out == nullptr) return MZGPU_E_INVALID;
  const ReduceIo io = reduce_io(shape, r);
  if (io.errs_rb && errs == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(r->ctx);
  MZ_TRY(reduce_io_check(io, shape, r, rows, out, errs));
  r->ctx->stats.rows_in += rows->ub;
  return reduce_step_dev(r, rows->mem.as<u64>(), buf_dlen(rows), rows->ub, upper, out, errs);
}

// The accumulable forms refuse a misuse without a message, and before a sticky context reports its own status.
extern "C" int32_t mzgpu_reduce_accumulable(mzgpu_reduce* r, const mzgpu_r32* rows, uint64_t n,
                                            int32_t mem, uint64_t upper, mzgpu_buf* out) {
  if (r == nullptr || out == nullptr || (rows == nullptr && n) || out->rb != 64 || r->shape != ReduceShape::ACCUM)
    return MZGPU_E_INVALID;
  return reduce_step(ReduceShape::ACCUM, r, rows, n, mem, upper, out, nullptr);
}
extern "C" int32_t mzgpu_reduce_accumulable_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper,
                                                mzgpu_buf* out) {
  if (r == nullptr || rows == nullptr || out == nullptr || rows->rb != 32 || out->rb != 64 ||
      r->shape != ReduceShape::ACCUM)
    return MZGPU_E_INVALID;
  return reduce_step_buf(ReduceShape::ACCUM, r, rows, upper, out, nullptr);
}
extern "C" int32_t mzgpu_reduce_lanes(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                                      mzgpu_buf* out) {
  return reduce_step(ReduceShape::LANES, r, rows, n, mem, upper, out, nullptr);
}
extern "C" int32_t mzgpu_reduce_lanes_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out) {
  return reduce_step_buf(ReduceShape::LANES, r, rows, upper, out, nullptr);
}
extern "C" int32_t mzgpu_reduce_monotonic(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                                          mzgpu_buf* out, mzgpu_buf* errs) {
  return reduce_step(ReduceShape::MONOTONIC, r, rows, n, mem, upper, out, errs);
}
extern "C" int32_t mzgpu_reduce_monotonic_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out,
                                              mzgpu_buf* errs) {
  return reduce_step_buf(ReduceShape::MONOTONIC, r, rows, upper, out, errs);
}
extern "C" int32_t mzgpu_reduce_hierarchical(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem,
                                             uint64_t upper, mzgpu_buf* out, mzgpu_buf* errs) {
  return reduce_step(ReduceShape::HIERARCHICAL, r, rows, n, mem, upper, out, errs);
}
extern "C" int32_t mzgpu_reduce_hierarchical_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out,
                                                 mzgpu_buf* errs) {
  return reduce_step_buf(ReduceShape::HIERARCHICAL, r, rows, upper, out, errs);
}
extern "C" int32_t mzgpu_topk_monotonic(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                                        mzgpu_buf* out, mzgpu_buf* errs) {
  return reduce_step(ReduceShape::TOPK_MONOTONIC, r, rows, n, mem, upper, out, errs);
}
extern "C" int32_t mzgpu_topk_monotonic_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out,
                                            mzgpu_buf* errs) {
  return reduce_step_buf(ReduceShape::TOPK_MONOTONIC, r, rows, upper, out, errs);
}
extern "C" int32_t mzgpu_topk_basic(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                                    mzgpu_buf* out, mzgpu_buf* errs) {
  return reduce_step(ReduceShape::TOPK_BASIC, r, rows, n, mem, upper, out, errs);
}
extern "C" int32_t mzgpu_topk_basic_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out,
                                        mzgpu_buf* errs) {
  return reduce_step_buf(ReduceShape::TOPK_BASIC, r, rows, upper, out, errs);
}

// ============================================================ Row keys as words (f1, first step)
extern "C" int32_t mzgpu_rowkey_pack(const uint8_t* row_bytes, uint64_t len, uint64_t* key_out) {
  if (key_out == nullptr || (row_bytes == nullptr && len)) return MZGPU_E_INVALID;
  if (len > 7) return MZGPU_E_UNSUPPORTED;
  u64 k = len << 56;
  for (u64 i = 0; i < len; ++i) k |= (u64)row_bytes[i] << (8 * (6 - i));
  *key_out = k;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_rowkeys_pack(const uint8_t* data, const uint64_t* offsets, uint64_t n, uint64_t* keys_out,
                                      uint64_t* n_done) {
  if ((n && (data == nullptr || offsets == nullptr || keys_out == nullptr))) return MZGPU_E_INVALID;
  for (u64 i = 0; i < n; ++i) {
    if (offsets[i + 1] < offsets[i]) return MZGPU_E_INVALID;
    const int32_t st = mzgpu_rowkey_pack(data + offsets[i], offsets[i + 1] - offsets[i], &keys_out[i]);
    if (st != MZGPU_OK) {
      if (n_done) *n_done = i;
      return st;
    }
  }
  if (n_done) *n_done = n;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_rowkey_unpack(uint64_t key, uint8_t row_bytes_out[7], uint64_t* len_out) {
  if (row_bytes_out == nullptr || len_out == nullptr) return MZGPU_E_INVALID;
  const u64 len = key >> 56;
  if (len > 7) return MZGPU_E_INVALID;
  for (u64 i = 0; i < len; ++i) row_bytes_out[i] = (uint8_t)(key >> (8 * (6 - i)));
  // canonical form: the padding below the row's bytes is zero
  if (len < 7 && (key & ((1ull << (8 * (7 - len))) - 1)) != 0) return MZGPU_E_INVALID;
  *len_out = len;
  return MZGPU_OK;
}

// ============================================================ correction buffer (f3)
struct mzgpu_correction {
  mzgpu_ctx* ctx;
  mzgpu_buf td;        // time-major rows (time, key, val | diff); sorted + consolidated iff !dirty
  u64 since = 0;       // Timestamp::MIN
  u64 applied = 0;     // the stored rows' times have been advanced to this
  bool dirty = false;  // rows were appended since the last consolidation
};
extern "C" int32_t mzgpu_correction_new(mzgpu_ctx* ctx, mzgpu_correction** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr) return MZGPU_E_INVALID;
  mzgpu_correction* c = new mzgpu_correction();
  c->ctx = ctx;
  c->td.ctx = ctx;
  c->td.rb = 32;
  buf_set_len(&c->td, 0);
  *out = c;
  return MZGPU_OK;
}
extern "C" void mzgpu_correction_free(mzgpu_correction* c) { delete c; }
static int32_t correction_insert_dev(mzgpu_correction* c, const u64* d_rows, DLen n, u64 n_ub, bool negate) {
  if (c->since == MZGPU_FRONTIER_EMPTY || n_ub == 0) return MZGPU_OK;  // the empty since discards everything
  mzgpu_ctx* ctx = c->ctx;
  MZ_TRY(buf_reserve(&c->td, c->td.ub + n_ub, true));
  Append a;
  MZ_TRY(buf_begin_append(&c->td, &a));
  MZ_TRY(mz_corr_to_td(ctx, d_rows, n, n_ub, c->since, negate, c->td.mem.as<u64>(), a.base, c->td.cap, a.out_len));
  buf_end_append(&c->td, a, n_ub);
  c->dirty = true;
  ctx->stats.rows_in += n_ub;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_correction_insert(mzgpu_correction* c, const mzgpu_r32* rows, uint64_t n, int32_t mem,
                                           int32_t negate) {
  if (c == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(c->ctx);
  if (n == 0) return MZGPU_OK;
  DevMem in;
  const u64* d_rows = (const u64*)rows;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(in.alloc(c->ctx, n * 32));
    MZ_TRY(copy_in(c->ctx, in.p, rows, n * 32, mem));
    d_rows = in.as<u64>();
  }
  return correction_insert_dev(c, d_rows, dlen_imm(n), n, negate != 0);
}
extern "C" int32_t mzgpu_correction_insert_buf(mzgpu_correction* c, mzgpu_buf* rows, int32_t negate) {
  if (c == nullptr || rows == nullptr || rows->rb != 32) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(c->ctx);
  return correction_insert_dev(c, rows->mem.as<u64>(), buf_dlen(rows), rows->ub, negate != 0);
}
// everything buffered: times advanced to `since`, sorted by (time, data), consolidated
static int32_t correction_consolidate(mzgpu_correction* c) {
  mzgpu_ctx* ctx = c->ctx;
  if (c->since == MZGPU_FRONTIER_EMPTY) {
    buf_set_len(&c->td, 0);
    c->dirty = false;
    return MZGPU_OK;
  }
  if (c->td.ub == 0 || (!c->dirty && c->applied == c->since)) return MZGPU_OK;
  if (c->applied != c->since) MZ_TRY(mz_corr_advance(ctx, c->td.mem.as<u64>(), buf_dlen(&c->td), c->td.ub, c->since));
  DevMem cons;
  u64 cap = 0;
  Lazy4 len;
  MZ_TRY(consolidate_dev(ctx, 32, c->td.mem.p, buf_dlen(&c->td), c->td.ub, &cons, &cap, &len));
  const u64 ub = len.known ? len.v[0] : c->td.ub;
  c->td.mem = std::move(cons);
  c->td.cap = cap;
  c->td.len = std::move(len);
  c->td.word = 0;
  c->td.ub = ub;
  c->applied = c->since;
  c->dirty = false;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_correction_updates_before(mzgpu_correction* c, uint64_t upper, mzgpu_buf* out) {
  if (c == nullptr || out == nullptr || out->rb != 32) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = c->ctx;
  MZ_CHECK_CTX(ctx);
  // PartialOrder::less_than(since, upper) on one-element antichains (correction_v2.rs:285)
  const bool since_lt_upper = c->since != MZGPU_FRONTIER_EMPTY && (upper == MZGPU_FRONTIER_EMPTY || c->since < upper);
  if (!since_lt_upper) return MZGPU_OK;
  MZ_TRY(correction_consolidate(c));
  if (c->td.ub == 0) return MZGPU_OK;
  Lazy4 cut;
  MZ_TRY(cut.make_pending(ctx));
  MZ_TRY(mz_corr_split(ctx, c->td.mem.as<u64>(), buf_dlen(&c->td), upper, cut.dptr()));
  cut.mark_written();
  MZ_TRY(buf_reserve(out, out->ub + c->td.ub, true));
  Append a;
  MZ_TRY(buf_begin_append(out, &a));
  MZ_TRY(mz_corr_from_td(ctx, c->td.mem.as<u64>(), dlen_of(cut, 0), c->td.ub, out->mem.as<u64>(), a.base, out->cap,
                         a.out_len));
  buf_end_append(out, a, c->td.ub);
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_correction_advance_since(mzgpu_correction* c, uint64_t since) {
  if (c == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(c->ctx);
  if (c->since != MZGPU_FRONTIER_EMPTY && since != MZGPU_FRONTIER_EMPTY && since < c->since) {
    MZ_SET_ERR(c->ctx, "correction: since regresses from %llu to %llu", (unsigned long long)c->since,
               (unsigned long long)since);
    return MZGPU_E_FRONTIER;
  }
  c->since = since;
  if (since == MZGPU_FRONTIER_EMPTY) {
    buf_set_len(&c->td, 0);
    c->dirty = false;
  }
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_correction_consolidate_at_since(mzgpu_correction* c) {
  if (c == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(c->ctx);
  return correction_consolidate(c);
}
extern "C" uint64_t mzgpu_correction_len(mzgpu_correction* c) {
  if (c == nullptr || c->ctx->sticky) return 0;
  if (correction_consolidate(c) != MZGPU_OK) return 0;
  if (buf_resolve(&c->td) != MZGPU_OK) return 0;
  return c->td.len.v[c->td.word];
}

// ====================================================== row L: linear join
// LinearJoinPlan rendered as linear_join.rs:230-527 does (see include/mzgpu.h): per stage a key
// preparation map, the "JoinStage" arrangement of the running result, and mz_join_core against
// the lookup arrangement.
struct mzgpu_linear_join {
  mzgpu_ctx* ctx = nullptr;
  mzgpu_linear_join_plan plan;
  uint32_t n = 0;
  mzgpu_spine* lookup[MZGPU_LINEAR_MAX_STAGES] = {};
  mzgpu_batcher* batcher[MZGPU_LINEAR_MAX_STAGES] = {};  // "JoinStage" arrange operators
  mzgpu_spine* stage[MZGPU_LINEAR_MAX_STAGES] = {};
  mzgpu_join* join[MZGPU_LINEAR_MAX_STAGES] = {};
  mzgpu_buf* keyed = nullptr;    // key-prepared rows of the stage being fed
  mzgpu_buf* running = nullptr;  // a stage's join output = the next stage's input
  mzgpu_buf* tmp = nullptr;
  u64 upper = 0;
  ~mzgpu_linear_join() {
    for (uint32_t s = 0; s < MZGPU_LINEAR_MAX_STAGES; ++s) {
      delete join[s];
      delete stage[s];
      delete batcher[s];
    }
    delete keyed;
    delete running;
    delete tmp;
  }
};
extern "C" int32_t mzgpu_linear_join_new(mzgpu_ctx* ctx, const mzgpu_linear_join_plan* plan,
                                         mzgpu_spine* const* lookup_traces, mzgpu_linear_join** out) {
  MZ_CHECK_CTX(ctx);
  if (plan == nullptr || lookup_traces == nullptr || out == nullptr) return MZGPU_E_INVALID;
  if (plan->n_stages == 0 || plan->n_stages > MZGPU_LINEAR_MAX_STAGES) {
    MZ_SET_ERR(ctx, "linear join: %u stages (1..%d supported)", plan->n_stages, MZGPU_LINEAR_MAX_STAGES);
    return MZGPU_E_UNSUPPORTED;
  }
  if (plan->has_initial_closure) MZ_TRY(validate_closure(ctx, &plan->initial_closure));
  if (plan->has_final_closure) MZ_TRY(validate_closure(ctx, &plan->final_closure));
  for (uint32_t s = 0; s < plan->n_stages; ++s) {
    if (lookup_traces[s] == nullptr || lookup_traces[s]->rb != 32 || lookup_traces[s]->ctx != ctx) return MZGPU_E_INVALID;
    MZ_TRY(validate_closure(ctx, &plan->stages[s].stream_key));
    MZ_TRY(validate_closure(ctx, &plan->stages[s].closure));
  }
  std::unique_ptr<mzgpu_linear_join> lj(new mzgpu_linear_join());
  lj->ctx = ctx;
  lj->plan = *plan;
  lj->n = plan->n_stages;
  for (mzgpu_buf** b : {&lj->keyed, &lj->running, &lj->tmp}) MZ_TRY(mzgpu_buf_new(ctx, 32, b));
  for (uint32_t s = 0; s < lj->n; ++s) {
    lj->lookup[s] = lookup_traces[s];
    MZ_TRY(mzgpu_batcher_new(ctx, 32, &lj->batcher[s]));
    MZ_TRY(mzgpu_spine_new(ctx, 32, 1, &lj->stage[s]));
    // join_core(stage arrangement, lookup arrangement): what the lookup trace already holds is
    // queued against the (empty) stage arrangement by the operator's pre-load (mz_join_core.rs:109-190)
    MZ_TRY(mzgpu_join_new(ctx, lj->stage[s], lj->lookup[s], &plan->stages[s].closure, &lj->join[s]));
  }
  *out = lj.release();
  return MZGPU_OK;
}
extern "C" void mzgpu_linear_join_free(mzgpu_linear_join* lj) { delete lj; }
extern "C" mzgpu_spine* mzgpu_linear_join_stage_trace(mzgpu_linear_join* lj, uint32_t stage) {
  return lj != nullptr && stage < lj->n ? lj->stage[stage] : nullptr;
}
extern "C" int32_t mzgpu_linear_join_step(mzgpu_linear_join* lj, mzgpu_buf* source,
                                          mzgpu_batch* const* lookup_batches, uint64_t upper, mzgpu_buf* out) {
  if (lj == nullptr || out == nullptr || out->rb != 32 || (source != nullptr && source->rb != 32) || source == out)
    return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = lj->ctx;
  MZ_CHECK_CTX(ctx);
  if (upper <= lj->upper) {
    MZ_SET_ERR(ctx, "linear join: frontier %llu does not advance past %llu", (unsigned long long)upper,
               (unsigned long long)lj->upper);
    return MZGPU_E_FRONTIER;
  }
  const u64 cap_time = lj->upper;  // the capability the join's outputs are produced under
  // the running result entering stage 0: the source updates behind the initial closure
  MZ_TRY(mzgpu_buf_clear(lj->running));
  if (source != nullptr && source->ub) {
    if (lj->plan.has_initial_closure)
      MZ_TRY(map_rows_into(ctx, source->mem.as<u64>(), buf_dlen(source), source->ub, &lj->plan.initial_closure,
                           MZGPU_FRONTIER_EMPTY, lj->running));
    else
      MZ_TRY(buf_append_dev(lj->running, source->mem.p, buf_dlen(source), source->ub));
  }
  for (uint32_t s = 0; s < lj->n; ++s) {
    // (a) LinearJoinKeyPreparation, (b) the JoinStage arrangement sealed at the new frontier
    MZ_TRY(mzgpu_buf_clear(lj->keyed));
    if (lj->running->ub)
      MZ_TRY(map_rows_into(ctx, lj->running->mem.as<u64>(), buf_dlen(lj->running), lj->running->ub,
                           &lj->plan.stages[s].stream_key, MZGPU_FRONTIER_EMPTY, lj->keyed));
    MZ_TRY(mzgpu_batcher_push_buf(lj->batcher[s], lj->keyed));
    mzgpu_batch* sb = nullptr;
    MZ_TRY(mzgpu_batcher_seal(lj->batcher[s], upper, &sb, nullptr));
    int32_t st = mzgpu_spine_insert(lj->stage[s], sb);
    // (c) mz_join_core over what is new on either side
    if (st == MZGPU_OK) st = mzgpu_join_core_push(lj->join[s], 0, sb, cap_time);
    mzgpu_batch_release(sb);
    MZ_TRY(st);
    if (lookup_batches != nullptr && lookup_batches[s] != nullptr)
      MZ_TRY(mzgpu_join_core_push(lj->join[s], 1, lookup_batches[s], cap_time));
    MZ_TRY(mzgpu_buf_clear(lj->tmp));
    int32_t done = 0;
    while (!done) MZ_TRY(mzgpu_join_core_work(lj->join[s], ~0ull, lj->tmp, &done));
    std::swap(lj->running, lj->tmp);
  }
  if (lj->running->ub) {
    if (lj->plan.has_final_closure)
      MZ_TRY(map_rows_into(ctx, lj->running->mem.as<u64>(), buf_dlen(lj->running), lj->running->ub,
                           &lj->plan.final_closure, MZGPU_FRONTIER_EMPTY, out));
    else
      MZ_TRY(buf_append_dev(out, lj->running->mem.p, buf_dlen(lj->running), lj->running->ub));
  }
  lj->upper = upper;
  return MZGPU_OK;
}

// ================================================ f4: columnar wire format
// Host side of column.cu: index arithmetic of `columnar::bytes::indexed`, the ship heuristic, and the
// entry points that move serialized containers in and out of row buffers.
static int col_slices(int32_t layout) {
  return layout == MZGPU_COLUMN_U64X2 ? 2 : layout == MZGPU_COLUMN_U64X4 ? 4 : layout == MZGPU_COLUMN_ROWROW ? 6 : 0;
}
static uint32_t col_row_bytes(int32_t layout) { return layout == MZGPU_COLUMN_U64X2 ? 16 : 32; }
static u64 col_words(int32_t layout, u64 rows, u64 kbytes, u64 vbytes) {
  switch (layout) {
    case MZGPU_COLUMN_U64X2: return 3 + 2 * rows;
    case MZGPU_COLUMN_U64X4: return 5 + 4 * rows;
    case MZGPU_COLUMN_ROWROW: return 7 + 4 * rows + (kbytes + 7) / 8 + (vbytes + 7) / 8;
  }
  return 0;
}
static bool col_at_capacity(u64 words) {
  const u64 ship = 1ull << 18;
  const u64 round = (words + (ship - 1)) & ~(ship - 1);
  return round - words < round / 10;
}
// word offsets of the slices of one container
static void col_offsets(int32_t layout, u64 rows, u64 kbytes, u64 vbytes, u64 off[6]) {
  const int k = col_slices(layout);
  u64 at = (u64)k + 1;
  for (int i = 0; i < 6; ++i) off[i] = 0;
  for (int i = 0; i < k; ++i) {
    off[i] = at;
    if (layout == MZGPU_COLUMN_ROWROW && i == 1)
      at += (kbytes + 7) / 8;
    else if (layout == MZGPU_COLUMN_ROWROW && i == 3)
      at += (vbytes + 7) / 8;
    else
      at += rows;
  }
}
extern "C" uint64_t mzgpu_column_length_in_words(int32_t layout, uint64_t rows, uint64_t key_bytes,
                                                 uint64_t val_bytes) {
  return col_words(layout, rows, key_bytes, val_bytes);
}
extern "C" int32_t mzgpu_column_at_capacity(uint64_t words) { return col_at_capacity(words) ? 1 : 0; }
extern "C" uint64_t mzgpu_column_ship_rows(int32_t layout) {
  if (layout != MZGPU_COLUMN_U64X2 && layout != MZGPU_COLUMN_U64X4) return 0;
  // the ship signal first fires at 2^18 - 2^18 / 10 + 1 words (the size grows by 2 or 4 words a push)
  const u64 ship = (1ull << 18) - (1ull << 18) / 10 + 1, per = layout == MZGPU_COLUMN_U64X2 ? 2 : 4;
  const u64 fixed = layout == MZGPU_COLUMN_U64X2 ? 3 : 5;
  return (ship - fixed + per - 1) / per;
}

extern "C" int32_t mzgpu_column_decode(mzgpu_ctx* ctx, int32_t layout, const uint64_t* words, uint64_t n_words,
                                       int32_t mem, mzgpu_buf* out) {
  MZ_CHECK_CTX(ctx);
  const int k = col_slices(layout);
  if (k == 0 || out == nullptr || words == nullptr || out->ctx != ctx || out->rb != col_row_bytes(layout) ||
      ((uintptr_t)words & 7))
    return MZGPU_E_INVALID;
  if (n_words < (u64)k + 1) {
    MZ_SET_ERR(ctx, "column_decode: %llu words cannot hold an index of %d offsets", (unsigned long long)n_words, k + 1);
    return MZGPU_E_INVALID;
  }
  u64 idx[7];
  if (mem == MZGPU_MEM_HOST) {
    std::memcpy(idx, words, 8 * (size_t)(k + 1));
  } else {
    MZ_CUDA(ctx, cudaMemcpyAsync(idx, words, 8 * (size_t)(k + 1), cudaMemcpyDeviceToHost, ctx->stream));
    MZ_SYNC(ctx);
  }
  // indexed::decode: slice i = [round_up(idx[i], 8), idx[i + 1]); a container of this layout has
  // k slices whose row-count-sized members agree
  bool ok = idx[0] == 8 * (u64)(k + 1) && idx[k] <= 8 * n_words;
  u64 off[6] = {0, 0, 0, 0, 0, 0}, len[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; ok && i < k; ++i) {
    const u64 lo = (idx[i] + 7) & ~7ull;
    if (idx[i + 1] < lo && !(idx[i + 1] == idx[i])) ok = false;
    off[i] = lo / 8;
    len[i] = idx[i + 1] >= lo ? idx[i + 1] - lo : 0;
  }
  const u64 n = ok ? len[k - 1] / 8 : 0;
  for (int i = 0; ok && i < k; ++i) {
    const bool bytes_slice = layout == MZGPU_COLUMN_ROWROW && (i == 1 || i == 3);
    if (!bytes_slice && len[i] != 8 * n) ok = false;
  }
  if (!ok) {
    MZ_SET_ERR(ctx, "column_decode: the index is not that of a layout-%d container", layout);
    return MZGPU_E_INVALID;
  }
  if (n == 0) return MZGPU_OK;
  DevMem in;
  const u64* d_words = words;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(in.alloc(ctx, n_words * 8));
    MZ_TRY(copy_in(ctx, in.p, words, n_words * 8, mem));
    d_words = in.as<u64>();
  }
  MZ_TRY(buf_resolve(out));  // the rows land at a base the host knows
  const u64 base = out->ub;
  MZ_TRY(buf_reserve(out, base + n, true));
  if (layout != MZGPU_COLUMN_ROWROW) {
    MZ_TRY(mz_col_decode_fixed(ctx, k, d_words, n, off, out->mem.as<u64>(), base));
    buf_set_len(out, base + n);
    ctx->stats.rows_in += n;
    return MZGPU_OK;
  }
  Lazy4 flag;
  MZ_TRY(flag.make_pending(ctx));
  MZ_CUDA(ctx, cudaMemsetAsync(flag.dptr(), 0, 32, ctx->stream));
  MZ_TRY(mz_col_decode_rows(ctx, d_words, n, off, len[1], len[3], out->mem.as<u64>(), base, flag.dptr()));
  flag.mark_written();
  MZ_TRY(flag.resolve());
  if (flag.v[0] == 2) {
    MZ_SET_ERR(ctx, "column_decode: Row bounds are not monotone or point outside the bytes slice");
    return MZGPU_E_INVALID;
  }
  if (flag.v[0] == 1) {
    MZ_SET_ERR(ctx, "column_decode: a Row is longer than 7 bytes (variable-width keys: SURVEY 8f-1)");
    return MZGPU_E_UNSUPPORTED;
  }
  buf_set_len(out, base + n);  // committed only now: a rejected container appends nothing
  ctx->stats.rows_in += n;
  return MZGPU_OK;
}

// prefix sums of the Row byte lengths of rows [first, first + n) (ROWROW)
struct RowPrefix {
  DevMem bsum, pk, pv;
  Lazy4 tot;
};
static int32_t row_prefix(mzgpu_ctx* ctx, const u64* d_rows, u64 first, u64 n, RowPrefix* rp) {
  const u64 nb = (n + 2047) / 2048;
  MZ_TRY(rp->bsum.alloc(ctx, 16 * (nb + 1)));
  MZ_TRY(rp->pk.alloc(ctx, 8 * (n + 1)));
  MZ_TRY(rp->pv.alloc(ctx, 8 * (n + 1)));
  MZ_TRY(rp->tot.make_pending(ctx));
  MZ_TRY(mz_col_row_prefix(ctx, d_rows, first, n, rp->bsum.as<u64>(), rp->pk.as<u64>(), rp->pv.as<u64>(),
                           rp->tot.dptr()));
  rp->tot.mark_written();
  return MZGPU_OK;
}
// one container of rows [s, s + n) of the range into d_words (capacity checked by the caller)
static int32_t col_encode_into(mzgpu_ctx* ctx, int32_t layout, const u64* d_rows, u64 first, u64 s, u64 n,
                               const RowPrefix* rp, u64 kbytes, u64 vbytes, u64* d_words) {
  u64 off[6];
  col_offsets(layout, n, kbytes, vbytes, off);
  if (layout != MZGPU_COLUMN_ROWROW) return mz_col_encode_fixed(ctx, col_slices(layout), d_rows, first + s, n, off, d_words);
  // zero padding of the two byte slices' last words
  if (kbytes % 8) MZ_CUDA(ctx, cudaMemsetAsync(d_words + off[1] + kbytes / 8, 0, 8, ctx->stream));
  if (vbytes % 8) MZ_CUDA(ctx, cudaMemsetAsync(d_words + off[3] + vbytes / 8, 0, 8, ctx->stream));
  return mz_col_encode_rows(ctx, d_rows, first, s, n, rp->pk.as<u64>(), rp->pv.as<u64>(), off, d_words);
}
// rows [first, first + n) of a device row array as ONE container in caller memory
static int32_t col_encode_range(mzgpu_ctx* ctx, int32_t layout, const u64* d_rows, u64 first, u64 n, u64* words,
                                u64 cap_words, int32_t mem, u64* n_words) {
  RowPrefix rp;
  u64 kb = 0, vb = 0;
  if (layout == MZGPU_COLUMN_ROWROW) {
    MZ_TRY(row_prefix(ctx, d_rows, first, n, &rp));
    MZ_TRY(rp.tot.resolve());
    kb = rp.tot.v[0], vb = rp.tot.v[1];
  }
  const u64 need = col_words(layout, n, kb, vb);
  if (n_words) *n_words = need;
  if (need > cap_words || words == nullptr) {
    MZ_SET_ERR(ctx, "column_encode: %llu words needed, capacity %llu", (unsigned long long)need,
               (unsigned long long)cap_words);
    return MZGPU_E_CAPACITY;
  }
  DevMem stage;
  u64* d_words = words;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(stage.alloc(ctx, need * 8));
    d_words = stage.as<u64>();
  }
  MZ_TRY(col_encode_into(ctx, layout, d_rows, first, 0, n, &rp, kb, vb, d_words));
  if (mem == MZGPU_MEM_HOST) MZ_TRY(copy_out(ctx, words, d_words, need * 8, mem));
  else MZ_SYNC(ctx);
  ctx->stats.rows_out += n;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_column_encode(mzgpu_buf* rows, int32_t layout, uint64_t first, uint64_t n, uint64_t* words,
                                       uint64_t cap_words, int32_t mem, uint64_t* n_words) {
  if (rows == nullptr || col_slices(layout) == 0 || rows->rb != col_row_bytes(layout) || ((uintptr_t)words & 7))
    return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = rows->ctx;
  MZ_CHECK_CTX(ctx);
  MZ_TRY(buf_resolve(rows));
  if (first > rows->ub) first = rows->ub;
  if (n > rows->ub - first) n = rows->ub - first;
  return col_encode_range(ctx, layout, rows->mem.as<u64>(), first, n, words, cap_words, mem, n_words);
}
extern "C" int32_t mzgpu_column_build(mzgpu_buf* rows, int32_t layout, uint64_t* words, uint64_t cap_words,
                                      int32_t mem, uint64_t* n_words, uint64_t* chunk_words, uint32_t cap_chunks,
                                      uint32_t* n_chunks) {
  if (rows == nullptr || col_slices(layout) == 0 || rows->rb != col_row_bytes(layout) || ((uintptr_t)words & 7))
    return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = rows->ctx;
  MZ_CHECK_CTX(ctx);
  MZ_TRY(buf_resolve(rows));
  const u64 n = rows->ub;
  // container j = rows [start[j], start[j + 1]) with kb[j] / vb[j] Row bytes
  std::vector<u64> ends, kbs, vbs;
  RowPrefix rp;
  if (layout != MZGPU_COLUMN_ROWROW) {
    const u64 ship = mzgpu_column_ship_rows(layout);
    for (u64 s = 0; s < n; s += ship) ends.push_back(std::min<u64>(n, s + ship));
    kbs.assign(ends.size(), 0), vbs.assign(ends.size(), 0);
  } else if (n) {
    MZ_TRY(row_prefix(ctx, rows->mem.as<u64>(), 0, n, &rp));
    const u64 cap = n / 39000 + 2;  // a container holds at least (235931 - 7) / 6 rows
    DevMem d_cuts;
    MZ_TRY(d_cuts.alloc(ctx, 8 * (3 * cap + 1)));
    MZ_TRY(mz_col_cuts(ctx, rp.pk.as<u64>(), rp.pv.as<u64>(), n, d_cuts.as<u64>() + 1, cap, d_cuts.as<u64>()));
    std::vector<u64> h(3 * cap + 1);
    MZ_TRY(copy_out(ctx, h.data(), d_cuts.p, 8 * h.size(), MZGPU_MEM_HOST));
    if (h[0] > cap) {
      MZ_SET_ERR(ctx, "column_build: %llu containers exceed the bound %llu", (unsigned long long)h[0], (unsigned long long)cap);
      return MZGPU_E_CAPACITY;
    }
    u64 pk = 0, pv = 0;
    for (u64 j = 0; j < h[0]; ++j) {
      ends.push_back(h[1 + 3 * j]);
      kbs.push_back(h[2 + 3 * j] - pk), vbs.push_back(h[3 + 3 * j] - pv);
      pk = h[2 + 3 * j], pv = h[3 + 3 * j];
    }
  }
  u64 total = 0;
  for (size_t j = 0; j < ends.size(); ++j) total += col_words(layout, ends[j] - (j ? ends[j - 1] : 0), kbs[j], vbs[j]);
  if (n_words) *n_words = total;
  if (n_chunks) *n_chunks = (uint32_t)ends.size();
  if (total > cap_words || ends.size() > cap_chunks || (total && words == nullptr) ||
      (!ends.empty() && chunk_words == nullptr)) {
    MZ_SET_ERR(ctx, "column_build: %llu words in %zu containers needed, capacity %llu / %u",
               (unsigned long long)total, ends.size(), (unsigned long long)cap_words, cap_chunks);
    return MZGPU_E_CAPACITY;
  }
  if (ends.empty()) return MZGPU_OK;
  DevMem stage;
  u64* d_words = words;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(stage.alloc(ctx, total * 8));
    d_words = stage.as<u64>();
  }
  u64 at = 0;
  for (size_t j = 0; j < ends.size(); ++j) {
    const u64 s = j ? ends[j - 1] : 0, cnt = ends[j] - s;
    MZ_TRY(col_encode_into(ctx, layout, rows->mem.as<u64>(), 0, s, cnt, &rp, kbs[j], vbs[j], d_words + at));
    chunk_words[j] = col_words(layout, cnt, kbs[j], vbs[j]);
    at += chunk_words[j];
  }
  if (mem == MZGPU_MEM_HOST) MZ_TRY(copy_out(ctx, words, d_words, total * 8, mem));
  else MZ_SYNC(ctx);
  ctx->stats.rows_out += n;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_batch_walk_column(mzgpu_batch* b, const uint64_t* key, uint64_t first, uint64_t fuel,
                                           int32_t layout, uint64_t* words, uint64_t cap_words, int32_t mem,
                                           uint64_t* n_words, uint64_t* n_rows) {
  if (b == nullptr || col_slices(layout) == 0 || b->rb != col_row_bytes(layout) || ((uintptr_t)words & 7))
    return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = b->ctx;
  MZ_CHECK_CTX(ctx);
  MZ_TRY(batch_ready(b));
  MZ_TRY(batch_resolve(b));
  u64 lo = 0, len = b->st.v[0];
  if (key != nullptr) {
    // seek_key: only this key's rows are walked (context.rs:1314-1333)
    mzgpu_key_run run;
    MZ_TRY(mzgpu_batch_seek_keys(b, key, 1, MZGPU_MEM_HOST, &run));
    if (run.len == 0 || run.key != *key) {
      lo = 0, len = 0;
    } else {
      lo = run.first, len = run.len;
    }
  }
  if (first > len) first = len;
  u64 cnt = len - first;
  if (cnt > fuel) cnt = fuel;
  if (n_rows) *n_rows = cnt;
  return col_encode_range(ctx, layout, b->rows.as<u64>(), lo + first, cnt, words, cap_words, mem, n_words);
}

// ================================================================= exchange
struct NcclId {
  char internal[128];
};
static void* open_nccl() {
  const char* names[] = {getenv("MZGPU_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    if (nm == nullptr) continue;
    void* h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    if (h) return h;
  }
  return nullptr;
}
extern "C" int32_t mzgpu_comm_unique_id(uint8_t id[MZGPU_COMM_ID_BYTES]) {
  void* lib = open_nccl();
  if (lib == nullptr) return MZGPU_E_NCCL;
  typedef int (*fn_t)(NcclId*);
  fn_t f = (fn_t)dlsym(lib, "ncclGetUniqueId");
  if (f == nullptr) return MZGPU_E_NCCL;
  NcclId uid;
  if (f(&uid) != 0) return MZGPU_E_NCCL;
  memcpy(id, uid.internal, MZGPU_COMM_ID_BYTES);
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_comm_init(mzgpu_ctx* ctx, const uint8_t id[MZGPU_COMM_ID_BYTES]) {
  MZ_CHECK_CTX(ctx);
  if (ctx->peers == 1) return MZGPU_OK;
  ctx->nccl_lib = open_nccl();
  if (ctx->nccl_lib == nullptr) {
    MZ_SET_ERR(ctx, "comm_init: cannot dlopen libnccl.so.2 (set MZGPU_NCCL_LIB)");
    return MZGPU_E_NCCL;
  }
  typedef int (*fn_t)(void**, int, NcclId, int);
  fn_t f = (fn_t)dlsym(ctx->nccl_lib, "ncclCommInitRank");
  if (f == nullptr) return MZGPU_E_NCCL;
  NcclId uid;
  memcpy(uid.internal, id, MZGPU_COMM_ID_BYTES);
  MZ_CUDA(ctx, cudaSetDevice(ctx->device));
  int rc = f(&ctx->nccl_comm, ctx->peers, uid, ctx->worker);
  if (rc != 0) {
    MZ_SET_ERR(ctx, "ncclCommInitRank failed with %d", rc);
    ctx->sticky = true;
    return MZGPU_E_NCCL;
  }
  return MZGPU_OK;
}

// k independent exchanges in one round: one partition per buffer, ONE counts
// all-to-all, ONE host wait (NCCL message sizes are host arguments), ONE payload
// all-to-all.  All peers must call with the same k (identical dataflows).
extern "C" int32_t mzgpu_exchange_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** ins, mzgpu_buf** outs) {
  MZ_CHECK_CTX(ctx);
  if (k == 0) return MZGPU_OK;
  if (ins == nullptr || outs == nullptr || k > MZ_MAX_EXCHANGE) return MZGPU_E_INVALID;
  for (uint32_t e = 0; e < k; ++e)
    if (ins[e] == nullptr || outs[e] == nullptr || ins[e]->rb != outs[e]->rb || ins[e] == outs[e])
      return MZGPU_E_INVALID;
  const u32 P = (u32)ctx->peers;
  if (P == 1) {
    for (uint32_t e = 0; e < k; ++e) {
      buf_set_len(outs[e], 0);
      MZ_TRY(buf_append_dev(outs[e], ins[e]->mem.p, buf_dlen(ins[e]), ins[e]->ub));
    }
    return MZGPU_OK;
  }
  if (ctx->nccl_comm == nullptr) {
    MZ_SET_ERR(ctx, "exchange: mzgpu_comm_init has not been called");
    return MZGPU_E_NCCL;
  }
  if (P > 16) {
    MZ_SET_ERR(ctx, "exchange: %u peers exceed the supported maximum 16", P);
    return MZGPU_E_UNSUPPORTED;
  }
  typedef int (*grp_t)();
  typedef int (*sr_t)(const void*, size_t, int, int, void*, cudaStream_t);
  typedef int (*rv_t)(void*, size_t, int, int, void*, cudaStream_t);
  static grp_t gstart = nullptr, gend = nullptr;
  static sr_t send = nullptr;
  static rv_t recv = nullptr;
  if (gstart == nullptr) {
    gstart = (grp_t)dlsym(ctx->nccl_lib, "ncclGroupStart");
    gend = (grp_t)dlsym(ctx->nccl_lib, "ncclGroupEnd");
    send = (sr_t)dlsym(ctx->nccl_lib, "ncclSend");
    recv = (rv_t)dlsym(ctx->nccl_lib, "ncclRecv");
  }
  if (!gstart || !gend || !send || !recv) return MZGPU_E_NCCL;
  const int NCCL_INT8 = 0, NCCL_UINT64 = 5;
#define NCCL_TRY(expr)                                        \
  do {                                                        \
    int _rc = (expr);                                         \
    if (_rc != 0) {                                           \
      MZ_SET_ERR(ctx, "NCCL call failed with %d at %s:%d", _rc, __FILE__, __LINE__); \
      ctx->sticky = true;                                     \
      return MZGPU_E_NCCL;                                    \
    }                                                         \
  } while (0)
  // 1. bucket rows by destination: counts and offsets stay on the device.
  // cnt layout: per exchange e: [e*P, e*P+P) send counts (contiguous over e so one
  // message per peer carries all k counts after the transpose below), cursors apart.
  DevMem parts[MZ_MAX_EXCHANGE], cnt;
  MZ_TRY(cnt.alloc(ctx, (size_t)(4 * MZ_MAX_EXCHANGE * 64) * 8));
  u64* d_cnt = cnt.as<u64>();                         // [e][64] send counts per exchange
  u64* d_cur = d_cnt + MZ_MAX_EXCHANGE * 64;          // [e][64] cursors
  u64* d_sendT = d_cur + MZ_MAX_EXCHANGE * 64;        // [p][k] send counts grouped by peer
  u64* d_recvT = d_sendT + MZ_MAX_EXCHANGE * 64;      // [p][k] recv counts grouped by peer
  {
    int rbs[MZ_MAX_EXCHANGE];
    const void* srcs[MZ_MAX_EXCHANGE];
    void* dsts[MZ_MAX_EXCHANGE];
    DLen ns[MZ_MAX_EXCHANGE];
    u64 ubs[MZ_MAX_EXCHANGE];
    for (uint32_t e = 0; e < k; ++e) {
      MZ_TRY(parts[e].alloc(ctx, std::max<u64>(ins[e]->ub, 1) * ins[e]->rb));
      rbs[e] = (int)ins[e]->rb;
      srcs[e] = ins[e]->mem.p;
      dsts[e] = parts[e].p;
      ns[e] = buf_dlen(ins[e]);
      ubs[e] = ins[e]->ub;
    }
    MZ_TRY(mz_partition_many(ctx, k, rbs, srcs, ns, ubs, P, dsts, d_cnt, d_cur, d_sendT));
  }
  // 2. counts all-to-all: k words per peer
  NCCL_TRY(gstart());
  for (u32 p = 0; p < P; ++p) {
    NCCL_TRY(send(d_sendT + (size_t)p * k, k, NCCL_UINT64, (int)p, ctx->nccl_comm, ctx->stream));
    NCCL_TRY(recv(d_recvT + (size_t)p * k, k, NCCL_UINT64, (int)p, ctx->nccl_comm, ctx->stream));
  }
  NCCL_TRY(gend());
  u64* h = ctx->h_big;  // pinned, 2 * 16 * MZ_MAX_EXCHANGE words
  MZ_CUDA(ctx, cudaMemcpyAsync(h, d_sendT, (size_t)P * k * 8, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_CUDA(ctx, cudaMemcpyAsync(h + 16 * MZ_MAX_EXCHANGE, d_recvT, (size_t)P * k * 8, cudaMemcpyDeviceToHost,
                               ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 2 * (size_t)P * k * 8;
  const u64* hs = h;
  const u64* hr = h + 16 * MZ_MAX_EXCHANGE;
  // 3. payload all-to-all
  u64 totals[MZ_MAX_EXCHANGE];
  for (uint32_t e = 0; e < k; ++e) {
    totals[e] = 0;
    for (u32 p = 0; p < P; ++p) totals[e] += hr[(size_t)p * k + e];
    buf_set_len(outs[e], 0);
    MZ_TRY(buf_reserve(outs[e], totals[e], false));
  }
  NCCL_TRY(gstart());
  for (uint32_t e = 0; e < k; ++e) {
    const u64 rb = ins[e]->rb;
    u64 soff = 0, roff = 0;
    for (u32 p = 0; p < P; ++p) {
      const u64 sc = hs[(size_t)p * k + e], rc = hr[(size_t)p * k + e];
      if (sc) NCCL_TRY(send((const char*)parts[e].p + soff * rb, sc * rb, NCCL_INT8, (int)p, ctx->nccl_comm, ctx->stream));
      if (rc) NCCL_TRY(recv((char*)outs[e]->mem.p + roff * rb, rc * rb, NCCL_INT8, (int)p, ctx->nccl_comm, ctx->stream));
      soff += sc;
      roff += rc;
    }
  }
  NCCL_TRY(gend());
  for (uint32_t e = 0; e < k; ++e) buf_set_len(outs[e], totals[e]);
  // `parts` are freed stream-ordered after the sends
  return MZGPU_OK;
#undef NCCL_TRY
}
// ---- exchange over peer memory (kernels in exchange.cu)
extern "C" int32_t mzgpu_comm_p2p_export(mzgpu_ctx* ctx, uint64_t landing_rows, uint32_t region_row_bytes,
                                         uint8_t handle[MZGPU_P2P_HANDLE_BYTES]) {
  MZ_CHECK_CTX(ctx);
  if (landing_rows == 0 || (region_row_bytes != 32 && region_row_bytes != 80) || ctx->peers > MZ_P2P_MAX_PEERS ||
      ctx->p2p_local != nullptr)
    return MZGPU_E_INVALID;
  const size_t bytes = mz_p2p_zone_bytes(landing_rows, region_row_bytes, (u32)ctx->peers);
  MZ_CUDA(ctx, cudaSetDevice(ctx->device));
  MZ_CUDA(ctx, cudaMalloc(&ctx->p2p_local, bytes));  // (not from the pool: the zone is exported)
  MZ_CUDA(ctx, cudaMemset(ctx->p2p_local, 0, MZ_P2P_HEADER_BYTES));
  MZ_CUDA(ctx, cudaMalloc((void**)&ctx->p2p_cursors, MZ_MAX_EXCHANGE * 16 * 8 + 16));
  MZ_CUDA(ctx, cudaMemset(ctx->p2p_cursors, 0, MZ_MAX_EXCHANGE * 16 * 8 + 16));
  ctx->p2p_done = (u32*)(ctx->p2p_cursors + MZ_MAX_EXCHANGE * 16);
  ctx->p2p_rows = landing_rows;
  ctx->p2p_region_rb = region_row_bytes;
  ctx->stats.device_bytes_in_use += bytes;
  if (ctx->stats.device_bytes_in_use > ctx->stats.device_bytes_peak) ctx->stats.device_bytes_peak = ctx->stats.device_bytes_in_use;
  if (handle != nullptr) {
    static_assert(sizeof(cudaIpcMemHandle_t) == MZGPU_P2P_HANDLE_BYTES, "IPC handle size");
    cudaIpcMemHandle_t h;
    MZ_CUDA(ctx, cudaIpcGetMemHandle(&h, ctx->p2p_local));
    memcpy(handle, &h, MZGPU_P2P_HANDLE_BYTES);
  }
  return MZGPU_OK;
}
extern "C" void* mzgpu_comm_p2p_zone(mzgpu_ctx* ctx) { return ctx ? ctx->p2p_local : nullptr; }
extern "C" int32_t mzgpu_comm_p2p_import(mzgpu_ctx* ctx, const uint8_t* handles) {
  MZ_CHECK_CTX(ctx);
  if (handles == nullptr || ctx->p2p_local == nullptr) return MZGPU_E_INVALID;
  MZ_CUDA(ctx, cudaSetDevice(ctx->device));
  for (int p = 0; p < ctx->peers; ++p) {
    if (p == ctx->worker) {
      ctx->p2p_peer[p] = ctx->p2p_local;
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)p * MZGPU_P2P_HANDLE_BYTES, MZGPU_P2P_HANDLE_BYTES);
    MZ_CUDA(ctx, cudaIpcOpenMemHandle(&ctx->p2p_peer[p], h, cudaIpcMemLazyEnablePeerAccess));
    ctx->p2p_peer_ipc[p] = true;
  }
  ctx->p2p_ready = true;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_comm_p2p_import_local(mzgpu_ctx* ctx, void* const* zones) {
  MZ_CHECK_CTX(ctx);
  if (zones == nullptr || ctx->p2p_local == nullptr) return MZGPU_E_INVALID;
  for (int p = 0; p < ctx->peers; ++p) {
    if (zones[p] == nullptr) return MZGPU_E_INVALID;
    ctx->p2p_peer[p] = zones[p];
  }
  if (ctx->p2p_peer[ctx->worker] != ctx->p2p_local) return MZGPU_E_INVALID;
  ctx->p2p_ready = true;
  return MZGPU_OK;
}
static int32_t p2p_check(mzgpu_ctx* ctx, uint32_t k) {
  if (k > MZ_MAX_EXCHANGE) return MZGPU_E_INVALID;
  if (!ctx->p2p_ready) {
    MZ_SET_ERR(ctx, "exchange_p2p: the landing zones have not been exported / imported");
    return MZGPU_E_INVALID;
  }
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_exchange_p2p_send(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** ins) {
  MZ_CHECK_CTX(ctx);
  if (k == 0) return MZGPU_OK;
  if (ins == nullptr) return MZGPU_E_INVALID;
  MZ_TRY(p2p_check(ctx, k));
  int rbs[MZ_MAX_EXCHANGE];
  const void* srcs[MZ_MAX_EXCHANGE];
  DLen ns[MZ_MAX_EXCHANGE];
  u64 ubs[MZ_MAX_EXCHANGE];
  for (uint32_t e = 0; e < k; ++e) {
    if (ins[e] == nullptr) return MZGPU_E_INVALID;
    rbs[e] = (int)ins[e]->rb;
    srcs[e] = ins[e]->mem.p;
    ns[e] = buf_dlen(ins[e]);
    ubs[e] = ins[e]->ub;
  }
  ctx->p2p_round++;
  return mz_p2p_send(ctx, k, rbs, srcs, ns, ubs);
}
extern "C" int32_t mzgpu_exchange_p2p_recv(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** outs, const uint64_t* recv_ub) {
  MZ_CHECK_CTX(ctx);
  if (k == 0) return MZGPU_OK;
  if (outs == nullptr) return MZGPU_E_INVALID;
  MZ_TRY(p2p_check(ctx, k));
  int rbs[MZ_MAX_EXCHANGE];
  void* dsts[MZ_MAX_EXCHANGE];
  u64 caps[MZ_MAX_EXCHANGE];
  u64* lens[MZ_MAX_EXCHANGE];
  const u64 most = (u64)ctx->peers * ctx->p2p_rows;
  for (uint32_t e = 0; e < k; ++e) {
    if (outs[e] == nullptr) return MZGPU_E_INVALID;
    u64 cap = recv_ub != nullptr && recv_ub[e] < most ? recv_ub[e] : most;
    if (cap == 0) cap = 1;
    buf_set_len(outs[e], 0);
    MZ_TRY(buf_reserve(outs[e], cap, false));
    MZ_TRY(outs[e]->len.make_pending(ctx));
    outs[e]->word = 0;
    outs[e]->ub = cap;
    rbs[e] = (int)outs[e]->rb;
    dsts[e] = outs[e]->mem.p;
    caps[e] = cap;
    lens[e] = outs[e]->len.dptr();
  }
  MZ_TRY(mz_p2p_recv(ctx, k, rbs, dsts, caps, lens));
  for (uint32_t e = 0; e < k; ++e) outs[e]->len.mark_written();
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_exchange_p2p(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** ins, mzgpu_buf** outs,
                                      const uint64_t* recv_ub) {
  MZ_CHECK_CTX(ctx);
  if (k == 0) return MZGPU_OK;
  if (ins == nullptr || outs == nullptr || k > MZ_MAX_EXCHANGE) return MZGPU_E_INVALID;
  for (uint32_t e = 0; e < k; ++e)
    if (ins[e] == nullptr || outs[e] == nullptr || ins[e]->rb != outs[e]->rb || ins[e] == outs[e])
      return MZGPU_E_INVALID;
  if (ctx->peers == 1) {
    for (uint32_t e = 0; e < k; ++e) {
      buf_set_len(outs[e], 0);
      MZ_TRY(buf_append_dev(outs[e], ins[e]->mem.p, buf_dlen(ins[e]), ins[e]->ub));
    }
    return MZGPU_OK;
  }
  MZ_TRY(mzgpu_exchange_p2p_send(ctx, k, ins));
  return mzgpu_exchange_p2p_recv(ctx, k, outs, recv_ub);
}

extern "C" int32_t mzgpu_partition_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf** ins, uint32_t peers,
                                        mzgpu_buf** outs, uint64_t* counts) {
  MZ_CHECK_CTX(ctx);
  if (k == 0) return MZGPU_OK;
  if (ins == nullptr || outs == nullptr || counts == nullptr || k > MZ_MAX_EXCHANGE || peers == 0 || peers > 64)
    return MZGPU_E_INVALID;
  for (uint32_t e = 0; e < k; ++e)
    if (ins[e] == nullptr || outs[e] == nullptr || ins[e]->rb != outs[e]->rb || ins[e] == outs[e])
      return MZGPU_E_INVALID;
  DevMem cnt;
  MZ_TRY(cnt.alloc(ctx, (size_t)(3 * MZ_MAX_EXCHANGE * 64) * 8));
  u64* d_cnt = cnt.as<u64>();
  u64* d_cur = d_cnt + MZ_MAX_EXCHANGE * 64;
  u64* d_sendT = d_cur + MZ_MAX_EXCHANGE * 64;
  int rbs[MZ_MAX_EXCHANGE];
  const void* srcs[MZ_MAX_EXCHANGE];
  void* dsts[MZ_MAX_EXCHANGE];
  DLen ns[MZ_MAX_EXCHANGE];
  u64 ubs[MZ_MAX_EXCHANGE];
  for (uint32_t e = 0; e < k; ++e) {
    buf_set_len(outs[e], 0);
    MZ_TRY(buf_reserve(outs[e], std::max<u64>(ins[e]->ub, 1), false));
    rbs[e] = (int)ins[e]->rb;
    srcs[e] = ins[e]->mem.p;
    dsts[e] = outs[e]->mem.p;
    ns[e] = buf_dlen(ins[e]);
    ubs[e] = ins[e]->ub;
  }
  MZ_TRY(mz_partition_many(ctx, k, rbs, srcs, ns, ubs, peers, dsts, d_cnt, d_cur, d_sendT));
  std::vector<u64> h((size_t)k * 64);
  MZ_TRY(copy_out(ctx, h.data(), d_cnt, h.size() * 8, MZGPU_MEM_HOST));
  for (uint32_t e = 0; e < k; ++e) {
    u64 tot = 0;
    for (uint32_t p = 0; p < peers; ++p) {
      counts[(size_t)e * peers + p] = h[(size_t)e * 64 + p];
      tot += h[(size_t)e * 64 + p];
    }
    buf_set_len(outs[e], tot);
  }
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_exchange(mzgpu_ctx* ctx, mzgpu_buf* in, mzgpu_buf* out) {
  return mzgpu_exchange_many(ctx, 1, &in, &out);
}

// ========================================================== temporal filter
// mzgpu_mfp_new (include/mzgpu.h): the device MfpPlan, and a BucketChain (src/timely-util/src/temporal.rs:59-211)
// of the updates it produced for future times.  A bucket [start, start + 2^bits) owns slices of device segments
// (mfp.cu); the host knows a bound on each slice's rows, and its exact size once the segment's header has been
// copied back.  Those copies are asynchronous into pinned memory and are read once the step that issued them has
// completed: the host never waits for them, except in mzgpu_mfp_frontier / mzgpu_mfp_stats.
struct MfpSeg {
  DevMem mem;  // MZ_MFP_HDR header words, then the rows
  u64 ub = 0;
  bool known = false;  // off[] holds the header
  u64 off[MZ_MFP_MAX_SLOTS + 1];
  int slot = -1;  // pinned mirror slot of the header copy in flight
  u64 seq = 0;    // the step that issued it
  u64* base() { return (u64*)mem.p; }
};
struct MfpSlice {
  std::shared_ptr<MfpSeg> seg;
  u32 idx;
};
static u64 mfp_slice_ub(const MfpSlice& s) {
  return s.seg->known ? s.seg->off[s.idx + 1] - s.seg->off[s.idx] : s.seg->ub;
}
// A bound on the rows of several slices: the slices of one segment whose header is not known yet together
// hold at most the segment's bound, however many of them there are.
static u64 mfp_slices_ub(const std::vector<MfpSlice>& v) {
  u64 known = 0;
  std::vector<std::pair<const MfpSeg*, u64>> unknown;
  for (const MfpSlice& s : v) {
    if (s.seg->known) {
      known += mfp_slice_ub(s);
      continue;
    }
    bool seen = false;
    for (auto& u : unknown) seen = seen || u.first == s.seg.get();
    if (!seen) unknown.emplace_back(s.seg.get(), s.seg->ub);
  }
  for (auto& u : unknown) known += u.second;
  return known;
}
struct MfpBucket {
  u32 bits;
  std::vector<MfpSlice> slices;
};
#define MZ_MFP_MIRROR 4096  // header copies in flight per operator
struct mzgpu_mfp_op {
  mzgpu_ctx* ctx;
  MfpDevPlan pl;
  int ow;
  u64 until;
  u64 upper = 0;
  std::map<u64, MfpBucket> chain;
  DevMem scratch;  // hist[65], cursor[65], touched, min time
  u64* h_mirror = nullptr;
  std::vector<int> free_slots;
  std::vector<std::shared_ptr<MfpSeg>> inflight;
  // held rows of earlier steps not in the chain yet: inserted at the next step (or read), once their header
  // copy has arrived, so that the insert is sized by the exact count rather than the step's bound
  std::vector<std::shared_ptr<MfpSeg>> pending;
  std::deque<std::pair<u64, cudaEvent_t>> events;
  u64 step_seq = 0, done_seq = 0;
  u64* hist() { return (u64*)scratch.p; }
  u64* touched() { return (u64*)scratch.p + 2 * MZ_MFP_MAX_SLOTS; }
  u64* dmin() { return (u64*)scratch.p + 2 * MZ_MFP_MAX_SLOTS + 1; }
  ~mzgpu_mfp_op() {
    inflight.clear();
    chain.clear();
    for (auto& e : events) cudaEventDestroy(e.second);
    if (h_mirror) cudaFreeHost(h_mirror);
  }
};

// bucket end (start + 2^bits), false when it is past u64::MAX (advance_by_power_of_two's None)
static bool mfp_bucket_end(u64 start, u32 bits, u64* end) {
  if (bits >= 64) return false;
  const u64 e = start + (1ull << bits);
  if (e < start || e == 0) return false;
  *end = e;
  return true;
}

// Read every header copy whose step has completed (wait = true: after waiting for the device, every one,
// and the headers never copied are read directly); drop empty slices.
static int32_t mfp_poll(mzgpu_mfp_op* op, bool wait) {
  mzgpu_ctx* ctx = op->ctx;
  if (wait) MZ_SYNC(ctx);
  while (!op->events.empty()) {
    const cudaError_t e = wait ? cudaSuccess : cudaEventQuery(op->events.front().second);
    if (e == cudaErrorNotReady) break;
    MZ_CUDA(ctx, e);
    op->done_seq = op->events.front().first;
    cudaEventDestroy(op->events.front().second);
    op->events.pop_front();
  }
  std::vector<std::shared_ptr<MfpSeg>> still;
  for (auto& s : op->inflight) {
    if (s->seq <= op->done_seq) {
      memcpy(s->off, op->h_mirror + (size_t)s->slot * MZ_MFP_HDR, sizeof(s->off));
      s->known = true;
      op->free_slots.push_back(s->slot);
      s->slot = -1;
    } else {
      still.push_back(std::move(s));
    }
  }
  op->inflight.swap(still);
  for (auto& kv : op->chain) {
    auto& v = kv.second.slices;
    if (wait)
      for (auto& sl : v)
        if (!sl.seg->known && sl.seg->slot < 0) {
          MZ_TRY(copy_out(ctx, sl.seg->off, sl.seg->base(), sizeof(sl.seg->off), MZGPU_MEM_HOST));
          sl.seg->known = true;
        }
    v.erase(std::remove_if(v.begin(), v.end(), [](const MfpSlice& s) { return s.seg->known && mfp_slice_ub(s) == 0; }),
            v.end());
  }
  return MZGPU_OK;
}

// Copy a segment's header back asynchronously (read by mfp_poll once the step has completed); with the pinned
// mirror full, the header stays unknown until a waiting call reads it.
static int32_t mfp_mirror(mzgpu_mfp_op* op, const std::shared_ptr<MfpSeg>& seg) {
  if (op->free_slots.empty()) return MZGPU_OK;
  mzgpu_ctx* ctx = op->ctx;
  seg->slot = op->free_slots.back();
  op->free_slots.pop_back();
  seg->seq = op->step_seq;
  MZ_CUDA(ctx, cudaMemcpyAsync(op->h_mirror + (size_t)seg->slot * MZ_MFP_HDR, seg->base(), sizeof(seg->off),
                               cudaMemcpyDeviceToHost, ctx->stream));
  op->inflight.push_back(seg);
  return MZGPU_OK;
}

// Partition the rows of `src` into the nb slots of a new segment (a row at time t goes to slot
// (# bounds <= t) - 1); *total, if set, gets its row count on the device.
static int32_t mfp_partition(mzgpu_mfp_op* op, const std::vector<MfpSlice>& src, const u64* bounds, u32 nb,
                             std::shared_ptr<MfpSeg>* out, u64* total, bool mirror) {
  mzgpu_ctx* ctx = op->ctx;
  const int nw = op->ow / 8;
  auto seg = std::make_shared<MfpSeg>();
  seg->ub = mfp_slices_ub(src);
  std::vector<MfpSlices> chunks;
  for (const MfpSlice& s : src) {
    if (mfp_slice_ub(s) == 0) continue;
    if (chunks.empty() || chunks.back().n == MZ_MFP_SLICES) {
      chunks.emplace_back();
      chunks.back().n = 0;
    }
    MfpSlices& c = chunks.back();
    c.base[c.n] = s.seg->base();
    c.idx[c.n] = s.idx;
    c.n++;
  }
  MZ_TRY(seg->mem.alloc(ctx, (MZ_MFP_HDR + seg->ub * (u64)nw) * 8));
  if (seg->ub == 0) {
    MZ_CUDA(ctx, cudaMemsetAsync(seg->mem.p, 0, MZ_MFP_HDR * 8, ctx->stream));
    if (total) MZ_CUDA(ctx, cudaMemsetAsync(total, 0, 8, ctx->stream));
    memset(seg->off, 0, sizeof(seg->off));
    seg->known = true;
  } else {
    MfpBounds b;
    memset(&b, 0, sizeof(b));
    b.nb = nb;
    for (u32 j = 0; j < nb; ++j) b.v[j] = bounds[j];
    MZ_TRY(mz_mfp_partition(ctx, op->ow, chunks.data(), (u32)chunks.size(), seg->ub, b, op->hist(),
                            op->hist() + MZ_MFP_MAX_SLOTS, seg->base(), total, op->touched()));
    if (mirror) MZ_TRY(mfp_mirror(op, seg));
  }
  *out = std::move(seg);
  return MZGPU_OK;
}

// BucketChain::split_and_insert: halve the bucket with a two-way time partition (no launch for an empty one)
static int32_t mfp_split(mzgpu_mfp_op* op, u64 start, MfpBucket&& bk, int64_t* fuel) {
  const u32 bits = bk.bits - 1;
  const u64 mid = start + (1ull << bits);
  MfpBucket lo{bits, {}}, hi{bits, {}};
  const u64 ub = mfp_slices_ub(bk.slices);
  if (ub > 0) {
    const u64 bnd[2] = {start, mid};
    std::shared_ptr<MfpSeg> seg;
    MZ_TRY(mfp_partition(op, bk.slices, bnd, 2, &seg, nullptr, true));
    lo.slices.push_back({seg, 0});
    hi.slices.push_back({seg, 1});
    *fuel -= (int64_t)ub;
  }
  op->chain[start] = std::move(lo);
  op->chain[mid] = std::move(hi);
  return MZGPU_OK;
}

// BucketChain::peel: the slices of every bucket below `upper`, splitting the one that straddles it
static int32_t mfp_peel(mzgpu_mfp_op* op, u64 upper, std::vector<MfpSlice>* peeled) {
  int64_t no_fuel = 0;
  while (!op->chain.empty()) {
    auto it = op->chain.begin();
    const u64 start = it->first;
    if (upper != MZGPU_FRONTIER_EMPTY && upper <= start) break;
    MfpBucket bk = std::move(it->second);
    op->chain.erase(it);
    u64 end = 0;
    const bool has_end = mfp_bucket_end(start, bk.bits, &end);
    if (upper != MZGPU_FRONTIER_EMPTY && (!has_end || upper < end)) {
      MZ_TRY(mfp_split(op, start, std::move(bk), &no_fuel));
    } else {
      for (auto& s : bk.slices) peeled->push_back(std::move(s));
    }
  }
  return MZGPU_OK;
}

// BucketChain::restore with fuel counted in rows (a split costs its bucket's row bound)
static int32_t mfp_restore(mzgpu_mfp_op* op) {
  int64_t fuel = MZGPU_MFP_RESTORE_FUEL;
  std::map<u64, MfpBucket> fresh;
  int64_t last = -2;
  while (fuel > 0 && !op->chain.empty()) {
    auto it = op->chain.begin();
    const u64 t = it->first;
    MfpBucket bk = std::move(it->second);
    op->chain.erase(it);
    if ((int64_t)bk.bits <= last + 2) {
      last = bk.bits;
      fresh.emplace(t, std::move(bk));
    } else {
      MZ_TRY(mfp_split(op, t, std::move(bk), &fuel));
    }
  }
  for (auto& kv : op->chain) fresh.emplace(kv.first, std::move(kv.second));
  op->chain.swap(fresh);
  return MZGPU_OK;
}

// the held rows of a step into the chain: rounds of up to 64 buckets, the rows past a round's last bucket in
// an overflow slot that the next round partitions again
static int32_t mfp_insert(mzgpu_mfp_op* op, MfpSlice held) {
  if (mfp_slice_ub(held) == 0) return MZGPU_OK;
  std::vector<MfpSlice> src{std::move(held)};
  auto it = op->chain.begin();
  while (it != op->chain.end()) {
    std::vector<MfpBucket*> bs;
    u64 bnd[MZ_MFP_MAX_SLOTS];
    u32 nb = 0;
    for (; it != op->chain.end() && nb < MZ_MFP_MAX_SLOTS - 1; ++it) {
      bnd[nb++] = it->first;
      bs.push_back(&it->second);
    }
    const u32 k = nb;
    if (it != op->chain.end()) bnd[nb++] = it->first;
    std::shared_ptr<MfpSeg> seg;
    MZ_TRY(mfp_partition(op, src, bnd, nb, &seg, nullptr, true));
    for (u32 j = 0; j < k; ++j) bs[j]->slices.push_back({seg, j});
    if (it == op->chain.end()) break;
    src.assign(1, MfpSlice{seg, k});
  }
  return MZGPU_OK;
}

// insert the held rows of earlier steps (their times are at least the upper they were evaluated at, which the
// chain still covers)
static int32_t mfp_flush_pending(mzgpu_mfp_op* op) {
  std::vector<std::shared_ptr<MfpSeg>> p;
  p.swap(op->pending);
  for (auto& seg : p) MZ_TRY(mfp_insert(op, {seg, 0}));
  return MZGPU_OK;
}

// the checks of a step, before it changes anything
static int32_t mfp_step_check(mzgpu_mfp_op* op, u64 upper, mzgpu_buf* out, mzgpu_buf* errs) {
  mzgpu_ctx* ctx = op->ctx;
  if (out == nullptr || errs == nullptr || out == errs || (int)out->rb != op->ow || errs->rb != 32) {
    MZ_SET_ERR(ctx, "mfp_step: out must hold %d-byte rows and errs 32-byte rows (distinct buffers)", op->ow);
    return MZGPU_E_INVALID;
  }
  if (upper < op->upper) {
    MZ_SET_ERR(ctx, "mfp_step: upper %llu is below the previous upper %llu", (unsigned long long)upper,
               (unsigned long long)op->upper);
    return MZGPU_E_FRONTIER;
  }
  return MZGPU_OK;
}

// A step's start: the held rows of earlier steps into the chain.
static int32_t mfp_step_begin(mzgpu_mfp_op* op) {
  MZ_TRY(mfp_poll(op, false));
  op->step_seq++;
  MZ_CUDA(op->ctx, cudaMemsetAsync(op->touched(), 0, 8, op->ctx->stream));
  return mfp_flush_pending(op);
}

// A step's end, once its new updates are in `ready` and `held` (bounds ub) and its errors in err_rows (count
// err_len on the device, bound err_ub): steps 2-6 below.
static int32_t mfp_step_end(mzgpu_mfp_op* op, const std::shared_ptr<MfpSeg>& ready, const std::shared_ptr<MfpSeg>& held,
                            const u64* err_rows, DLen err_len, u64 err_ub, u64 upper, mzgpu_buf* out,
                            mzgpu_buf* errs) {
  mzgpu_ctx* ctx = op->ctx;
  // 2. peel the due buckets; 3. release them with the ready rows, consolidated
  std::vector<MfpSlice> rel;
  MZ_TRY(mfp_peel(op, upper, &rel));
  rel.push_back({ready, 0});
  if (mfp_slices_ub(rel) > 0) {
    Lazy4 tot;
    MZ_TRY(tot.make_pending(ctx));
    std::shared_ptr<MfpSeg> all;
    const u64 zero = 0;
    MZ_TRY(mfp_partition(op, rel, &zero, 1, &all, tot.dptr(), false));
    tot.mark_written();
    MZ_TRY(append_consolidated(ctx, op->ow, all->base() + MZ_MFP_HDR, dlen_of(tot, 0), all->ub, out));
  }
  rel.clear();
  // 4. restore the chain; 5. hold the rest (inserted by the next step or read)
  MZ_TRY(mfp_restore(op));
  if (held->ub > 0) {
    MZ_TRY(mfp_mirror(op, held));
    op->pending.push_back(held);
  }
  // 6. errors
  if (err_ub > 0) MZ_TRY(append_consolidated(ctx, 32, err_rows, err_len, err_ub, errs));
  cudaEvent_t ev;
  MZ_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  MZ_CUDA(ctx, cudaEventRecord(ev, ctx->stream));
  op->events.emplace_back(op->step_seq, ev);
  op->upper = upper;
  return MZGPU_OK;
}

// ready / held segments for up to `ub` updates (empty and known when ub == 0), their counts zeroed
static int32_t mfp_segments(mzgpu_mfp_op* op, u64 ub, std::shared_ptr<MfpSeg>* ready, std::shared_ptr<MfpSeg>* held) {
  mzgpu_ctx* ctx = op->ctx;
  *ready = std::make_shared<MfpSeg>();
  *held = std::make_shared<MfpSeg>();
  for (MfpSeg* s : {ready->get(), held->get()}) {
    s->ub = ub;
    if (ub > 0) {
      MZ_TRY(s->mem.alloc(ctx, (MZ_MFP_HDR + ub * (u64)(op->ow / 8)) * 8));
      MZ_CUDA(ctx, cudaMemsetAsync(s->mem.p, 0, 16, ctx->stream));
    } else {
      s->known = true;
      memset(s->off, 0, sizeof(s->off));
    }
  }
  return MZGPU_OK;
}

static int32_t mfp_step_dev(mzgpu_mfp_op* op, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                            mzgpu_buf* errs) {
  mzgpu_ctx* ctx = op->ctx;
  MZ_TRY(mfp_step_check(op, upper, out, errs));
  MZ_TRY(mfp_step_begin(op));
  // 1. evaluate the new rows: ready, held and error rows
  std::shared_ptr<MfpSeg> ready, held;
  MZ_TRY(mfp_segments(op, 2 * n_ub, &ready, &held));
  DevMem err_rows;
  Lazy4 err_len;
  if (n_ub > 0) {
    MZ_TRY(err_rows.alloc(ctx, n_ub * 32));
    MZ_TRY(err_len.make_pending(ctx));
    MZ_CUDA(ctx, cudaMemsetAsync(err_len.dptr(), 0, 8, ctx->stream));
    MZ_TRY(mz_mfp_eval(ctx, op->pl, d_rows, n, n_ub, upper, op->until, ready->base(), held->base(),
                       (u64*)err_rows.p, err_len.dptr()));
    err_len.mark_written();
  }
  return mfp_step_end(op, ready, held, (const u64*)err_rows.p, n_ub > 0 ? dlen_of(err_len, 0) : dlen_imm(0), n_ub,
                      upper, out, errs);
}

// The checks of one program (include/mzgpu.h): a type per stack slot, simulated op by op, and whether the slot may
// carry an error whose payload varies with the data (kept out of AND / OR).  MZGPU_E_INVALID is returned at once; a
// well-formed construct outside the subset is noted in *unsupported (the first one).
enum MfpTy { MFP_INT32, MFP_INT64, MFP_BOOL, MFP_MZTS, MFP_TS, MFP_DATE };
enum MfpKind { MFP_PREDICATE, MFP_TEMPORAL, MFP_MAP };
struct MfpProgram {
  MfpKind kind;
  uint32_t index;  // predicate / temporal predicate / expression number
  const mzgpu_having_op* ops;
  uint32_t n_ops;
  const mzgpu_having_const* consts;  // the program's constant pool
  uint32_t n_consts;
  i64* iv_us;                // its folded intervals
  const MfpTy* map_ty;       // the types of the expressions it may read: [0, n_readable)
  uint32_t n_readable;
  uint32_t n_fn;             // FlatMap extension columns it may read (MZGPU_SRC_FN0 + i, i < n_fn)
};
static int32_t validate_mfp_program(mzgpu_ctx* ctx, uint32_t in_row_bytes, const MfpProgram& g, MfpTy* result,
                                    uint32_t* support, const char** unsupported) {
  const char* what = g.kind == MFP_TEMPORAL ? "temporal predicate" : g.kind == MFP_MAP ? "expression" : "predicate";
  const bool predicate = g.kind == MFP_PREDICATE;
  auto bad = [&](uint32_t i, const char* why) {
    MZ_SET_ERR(ctx, "mfp: %s %u, op %u: %s", what, g.index, i, why);
    return MZGPU_E_INVALID;
  };
  auto outside = [&](uint32_t i, const char* why) {
    if (*unsupported == nullptr) {
      MZ_SET_ERR(ctx, "mfp: %s %u, op %u: %s", what, g.index, i, why);
      *unsupported = why;
    }
  };
  const uint32_t max_src = in_row_bytes == 40 ? MZGPU_SRC_VAL2 : MZGPU_SRC_VAL1;
  if (g.n_ops == 0 || g.n_ops > MZGPU_MFP_MAX_OPS) return bad(0, "op count (1..16)");
  MfpTy ty[MZGPU_HAVING_MAX_STACK];
  bool varying[MZGPU_HAVING_MAX_STACK];
  int sp = 0;
  *support = 0;
  for (uint32_t i = 0; i < g.n_ops; ++i) {
    const mzgpu_having_op& o = g.ops[i];
    const uint32_t code = o.code;
    const bool col = code == MZGPU_HOP_COL || code == MZGPU_HOP_COL_MZTS || code == MZGPU_HOP_COL_TS ||
                     code == MZGPU_HOP_COL_DATE || code == MZGPU_HOP_COL_F64;
    if (col || code == MZGPU_HOP_INT || code == MZGPU_HOP_MAP) {
      if (sp == MZGPU_HAVING_MAX_STACK) return bad(i, "stack overflow (depth 8)");
      MfpTy t = MFP_INT64;
      if (col) {
        if (o.arg > max_src && !(o.arg >= MZGPU_SRC_FN0 && o.arg < MZGPU_SRC_FN0 + g.n_fn))
        return bad(i, "column word out of range");
        if (o.bits == 0 || o.bits > 64 || (uint32_t)o.shift + o.bits > 64 || o.sign_extend > 1)
          return bad(i, "column field is empty or out of range");
        if (code == MZGPU_HOP_COL) t = (o.bits < 32 || (o.bits == 32 && o.sign_extend)) ? MFP_INT32 : MFP_INT64;
        if (code == MZGPU_HOP_COL_MZTS) {
          if (o.sign_extend) return bad(i, "an mz_timestamp column is unsigned");
          t = MFP_MZTS;
        }
        if (code == MZGPU_HOP_COL_TS) t = MFP_TS;
        if (code == MZGPU_HOP_COL_DATE) {
          if (o.bits > 32 || (o.bits == 32 && !o.sign_extend)) return bad(i, "a date column is at most an i32");
          t = MFP_DATE;
        }
        if (code == MZGPU_HOP_COL_F64) {
          if (o.bits != 64) return bad(i, "a float64 column is a whole word");
          outside(i, "float64 columns");
        }
      } else if (code == MZGPU_HOP_MAP) {
        if (o.arg >= g.n_readable)
          return bad(i, g.kind == MFP_MAP ? "reads an expression at or after its own" : "expression index out of range");
        t = g.map_ty[o.arg];
        if (o.arg + 1u > *support) *support = o.arg + 1u;
      } else {
        if (o.konst >= g.n_consts) return bad(i, "constant index out of range");
        const mzgpu_having_const& k = g.consts[o.konst];
        if (k.hi != ((int64_t)k.lo < 0 ? ~0ull : 0ull)) return bad(i, "INT constant outside i64");
        t = (int64_t)k.lo >= INT32_MIN && (int64_t)k.lo <= INT32_MAX ? MFP_INT32 : MFP_INT64;
      }
      if (predicate && (t == MFP_MZTS || t == MFP_TS || t == MFP_DATE))
        outside(i, "mz_timestamp values in a non-temporal predicate");
      varying[sp] = false;  // an expression read here has been evaluated without error
      ty[sp++] = t;
      continue;
    }
    const bool unary_int = code == MZGPU_HOP_NEG || code == MZGPU_HOP_ABS || code == MZGPU_HOP_INT64_TO_INT32;
    if ((code >= MZGPU_HOP_INT_TO_MZTS && code <= MZGPU_HOP_DATE_TO_MZTS) || unary_int) {  // (COL_TS / COL_DATE above)
      if (sp < 1) return bad(i, "stack underflow");
      MfpTy& a = ty[sp - 1];
      const bool ia = a == MFP_INT32 || a == MFP_INT64;
      if (unary_int) {
        if (!ia) return bad(i, "integer function of a non-integer");
        if (code == MZGPU_HOP_INT64_TO_INT32) {
          a = MFP_INT32;
          varying[sp - 1] = true;  // Int32OutOfRange carries the operand
        } else {
          if (o.arg != 32 && o.arg != 64) return bad(i, "width is not 32 or 64");
          if (o.arg == 32 && a != MFP_INT32) return bad(i, "32-bit operation on an operand that is not int32");
          a = o.arg == 32 ? MFP_INT32 : MFP_INT64;
        }
        continue;
      }
      if (code == MZGPU_HOP_INT_TO_MZTS) {
        if (!ia) return bad(i, "cast to mz_timestamp of a non-integer");
        a = MFP_MZTS;
        varying[sp - 1] = true;
      } else if (code == MZGPU_HOP_TS_TO_MZTS) {
        if (a != MFP_TS) return bad(i, "timestamp cast of a non-timestamp");
        a = MFP_MZTS;
        varying[sp - 1] = true;
      } else if (code == MZGPU_HOP_DATE_TO_MZTS) {
        if (a != MFP_DATE) return bad(i, "date cast of a non-date");
        a = MFP_MZTS;
        varying[sp - 1] = true;
      } else {  // MZGPU_HOP_TS_ADD_IV
        if (a != MFP_TS) return bad(i, "interval added to a non-timestamp");
        if (o.konst >= g.n_consts) return bad(i, "constant index out of range");
        const mzgpu_having_const& k = g.consts[o.konst];
        const int32_t days = (int32_t)(uint32_t)k.hi, months = (int32_t)(uint32_t)(k.hi >> 32);
        const __int128 us = (__int128)days * 86400000000ll + (__int128)(int64_t)k.lo;
        if (months != 0) outside(i, "intervals with months");
        else if (us < (__int128)INT64_MIN || us > (__int128)INT64_MAX) outside(i, "interval beyond i64 microseconds");
        else g.iv_us[o.konst] = (i64)us;
      }
      if (predicate) outside(i, "mz_timestamp values in a non-temporal predicate");
      continue;
    }
    if (code == MZGPU_HOP_NOT) {
      if (sp < 1) return bad(i, "stack underflow");
      if (ty[sp - 1] != MFP_BOOL) return bad(i, "NOT of a non-BOOL");
      continue;
    }
    if (code == MZGPU_HOP_IF) {
      if (sp < 3) return bad(i, "stack underflow");
      const MfpTy c = ty[sp - 3], t = ty[sp - 2], e = ty[sp - 1];
      const bool it = t == MFP_INT32 || t == MFP_INT64, ie = e == MFP_INT32 || e == MFP_INT64;
      if (c != MFP_BOOL) return bad(i, "IF on a non-BOOL condition");
      if (t != e && !(it && ie)) return bad(i, "IF branches of different types");
      ty[sp - 3] = t == e ? t : MFP_INT64;
      varying[sp - 3] = varying[sp - 3] || varying[sp - 2] || varying[sp - 1];
      sp -= 2;
      continue;
    }
    const bool arith = (code >= MZGPU_HOP_ADD && code <= MZGPU_HOP_DIV) || code == MZGPU_HOP_MOD;
    if (!arith && code != MZGPU_HOP_CMP && code != MZGPU_HOP_AND && code != MZGPU_HOP_OR) return bad(i, "unknown opcode");
    if (sp < 2) return bad(i, "stack underflow");
    const MfpTy a = ty[sp - 2], b = ty[sp - 1];
    const bool va = varying[sp - 2], vb = varying[sp - 1];
    --sp;
    const bool ia = a == MFP_INT32 || a == MFP_INT64, ib = b == MFP_INT32 || b == MFP_INT64;
    varying[sp - 1] = va || vb;
    if (code == MZGPU_HOP_AND || code == MZGPU_HOP_OR) {
      if (a != MFP_BOOL || b != MFP_BOOL) return bad(i, "AND / OR of a non-BOOL");
      if (va || vb) outside(i, "AND / OR over an error whose payload varies with the data");
    } else if (code == MZGPU_HOP_CMP) {
      if (o.arg > MZGPU_CMP_GE) return bad(i, "unknown compare op");
      if ((a == MFP_BOOL) != (b == MFP_BOOL)) return bad(i, "BOOL compared with a value");
      if (a == MFP_BOOL) outside(i, "BOOL comparisons");
      else if (!ia || !ib) outside(i, "comparisons of mz_timestamp, timestamp or date values");
      ty[sp - 1] = MFP_BOOL;
    } else {
      if (o.arg != 32 && o.arg != 64) return bad(i, "width is not 32 or 64");
      if (!ia || !ib) return bad(i, "arithmetic on a non-integer");
      if (o.arg == 32 && (a != MFP_INT32 || b != MFP_INT32))
        return bad(i, "32-bit operation on an operand that is not int32");
      ty[sp - 1] = o.arg == 32 ? MFP_INT32 : MFP_INT64;
    }
  }
  if (g.kind == MFP_MAP) {
    if (sp != 1) return bad(g.n_ops, "the expression does not leave one value");
  } else if (sp != 1 || ty[0] != (g.kind == MFP_TEMPORAL ? MFP_MZTS : MFP_BOOL)) {
    return bad(g.n_ops, g.kind == MFP_TEMPORAL ? "the program does not leave one mz_timestamp"
                                               : "the predicate does not leave one BOOL");
  }
  *result = ty[0];
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_mfp_new(mzgpu_ctx* ctx, const mzgpu_mfp* plan, uint64_t until, mzgpu_mfp_op** out) {
  return mzgpu_mfp_new_map(ctx, plan, nullptr, until, out);
}

// The plan of mzgpu_mfp_new_map, checked, over input rows with n_fn FlatMap extension columns.
static int32_t mfp_build_plan(mzgpu_ctx* ctx, const mzgpu_mfp* plan, const mzgpu_mfp_map* map, uint32_t n_fn,
                              MfpDevPlan* out_pl) {
  if (plan == nullptr) return MZGPU_E_INVALID;
  const mzgpu_mfp& m = *plan;
  if (map != nullptr && map->n_exprs == 0) map = nullptr;  // exactly mzgpu_mfp_new
  if ((m.in_row_bytes != 32 && m.in_row_bytes != 40) || (m.out_row_bytes != 32 && m.out_row_bytes != 40)) {
    MZ_SET_ERR(ctx, "mfp: rows are 32 or 40 bytes (in %u, out %u)", m.in_row_bytes, m.out_row_bytes);
    return MZGPU_E_INVALID;
  }
  if (m.n_predicates > MZGPU_MFP_MAX_PREDICATES || m.n_temporal > MZGPU_MFP_MAX_TEMPORAL ||
      m.n_consts > MZGPU_MFP_MAX_CONSTS) {
    MZ_SET_ERR(ctx, "mfp: %u predicates (0..4), %u temporal predicates (0..4), %u constants (0..8)", m.n_predicates,
               m.n_temporal, m.n_consts);
    return MZGPU_E_INVALID;
  }
  if (map && (map->n_exprs > MZGPU_MFP_MAX_MAPS || map->n_consts > MZGPU_MFP_MAX_CONSTS)) {
    MZ_SET_ERR(ctx, "mfp: %u expressions (0..8), %u expression constants (0..8)", map->n_exprs, map->n_consts);
    return MZGPU_E_INVALID;
  }
  const uint32_t n_exprs = map ? map->n_exprs : 0;
  const uint32_t max_src = m.in_row_bytes == 40 ? MZGPU_SRC_VAL2 : MZGPU_SRC_VAL1;
  for (int k = 0; k < 3; ++k) {
    if (m.n_fields[k] > MZGPU_MAX_FIELDS || (k == 2 && m.out_row_bytes == 32 && m.n_fields[2] != 0)) {
      MZ_SET_ERR(ctx, "mfp: %u fields for output word %d", m.n_fields[k], k);
      return MZGPU_E_INVALID;
    }
    for (uint32_t f = 0; f < m.n_fields[k]; ++f) {
      mzgpu_field fd = m.fields[k][f];
      const bool is_map = fd.src >= MZGPU_SRC_MAP0;
      if (is_map && fd.src - MZGPU_SRC_MAP0 >= n_exprs) {
        MZ_SET_ERR(ctx, "mfp: output word %d, field %u reads expression %u of %u", k, f, fd.src - MZGPU_SRC_MAP0,
                   n_exprs);
        return MZGPU_E_INVALID;
      }
      const bool is_fn = fd.src >= MZGPU_SRC_FN0 && fd.src < MZGPU_SRC_FN0 + n_fn;
      if (is_map || is_fn) fd.src = MZGPU_SRC_KEY;  // the bit-field checks of an input field
      MZ_TRY(validate_field(ctx, fd, true));
      if ((!is_map && fd.src > max_src) || (uint32_t)fd.shift + fd.bits > 64) {
        MZ_SET_ERR(ctx, "mfp: output word %d, field %u reads past the input row", k, f);
        return MZGPU_E_INVALID;
      }
    }
  }
  MfpDevPlan pl;
  memset(&pl, 0, sizeof(pl));
  pl.plan = m;
  if (map) pl.map = *map;
  const char* unsupported = nullptr;
  std::string unsupported_msg;
  MfpTy map_ty[MZGPU_MFP_MAX_MAPS];
  for (uint32_t e = 0; e < n_exprs; ++e) {
    const MfpProgram g{MFP_MAP, e, map->ops[e], map->n_ops[e], map->consts, map->n_consts, pl.map_iv_us, map_ty, e,
                       n_fn};
    uint32_t support;
    MZ_TRY(validate_mfp_program(ctx, m.in_row_bytes, g, &map_ty[e], &support, &unsupported));
    if (unsupported && unsupported_msg.empty()) unsupported_msg = ctx->last_error;
  }
  for (uint32_t p = 0; p < m.n_predicates; ++p) {
    const MfpProgram g{MFP_PREDICATE, p, m.ops[p], m.n_ops[p], m.consts, m.n_consts, pl.iv_us, map_ty, n_exprs,
                       n_fn};
    MfpTy t;
    MZ_TRY(validate_mfp_program(ctx, m.in_row_bytes, g, &t, &pl.support[p], &unsupported));
    if (unsupported && unsupported_msg.empty()) unsupported_msg = ctx->last_error;
  }
  for (uint32_t p = 0; p < m.n_temporal; ++p) {
    const uint32_t c = m.temporal_cmp[p];
    if (c > MZGPU_CMP_GE) {
      MZ_SET_ERR(ctx, "mfp: temporal predicate %u: unknown compare op %u", p, c);
      return MZGPU_E_INVALID;
    }
    if (c == MZGPU_CMP_NE && unsupported == nullptr) {
      MZ_SET_ERR(ctx, "mfp: temporal predicate %u: mz_now() <> expr is not a temporal filter", p);
      unsupported = "<>";
    }
    const MfpProgram g{MFP_TEMPORAL, p, m.temporal_ops[p], m.n_temporal_ops[p], m.consts, m.n_consts, pl.iv_us,
                       map_ty, n_exprs, n_fn};
    MfpTy t;
    uint32_t support;
    MZ_TRY(validate_mfp_program(ctx, m.in_row_bytes, g, &t, &support, &unsupported));
    if (unsupported && unsupported_msg.empty()) unsupported_msg = ctx->last_error;
    // MfpPlan::create_from (src/expr/src/linear.rs:1772-1804)
    if (c == MZGPU_CMP_EQ) {
      pl.lower[pl.n_lower++] = p;
      pl.upper[pl.n_upper++] = p | 8;
    } else if (c == MZGPU_CMP_LT) {
      pl.upper[pl.n_upper++] = p;
    } else if (c == MZGPU_CMP_LE) {
      pl.upper[pl.n_upper++] = p | 8;
    } else if (c == MZGPU_CMP_GT) {
      pl.lower[pl.n_lower++] = p | 8;
    } else if (c == MZGPU_CMP_GE) {
      pl.lower[pl.n_lower++] = p;
    }
  }
  if (unsupported) {
    ctx->last_error = unsupported_msg;
    return MZGPU_E_UNSUPPORTED;
  }
  *out_pl = pl;
  return MZGPU_OK;
}

static int32_t mfp_op_create(mzgpu_ctx* ctx, const MfpDevPlan& pl, uint64_t until,
                             std::unique_ptr<mzgpu_mfp_op>* out) {
  auto op = std::unique_ptr<mzgpu_mfp_op>(new mzgpu_mfp_op());
  op->ctx = ctx;
  op->pl = pl;
  op->ow = (int)pl.plan.out_row_bytes;
  op->until = until;
  MZ_TRY(op->scratch.alloc(ctx, (2 * MZ_MFP_MAX_SLOTS + 2) * 8));
  MZ_CUDA(ctx, cudaMemsetAsync(op->scratch.p, 0, (2 * MZ_MFP_MAX_SLOTS + 2) * 8, ctx->stream));
  MZ_CUDA(ctx, cudaMallocHost((void**)&op->h_mirror, (size_t)MZ_MFP_MIRROR * MZ_MFP_HDR * 8));
  for (int s = MZ_MFP_MIRROR - 1; s >= 0; --s) op->free_slots.push_back(s);
  op->chain.emplace(0, MfpBucket{64, {}});  // BucketChain::new: one bucket over the whole domain
  *out = std::move(op);
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_mfp_new_map(mzgpu_ctx* ctx, const mzgpu_mfp* plan, const mzgpu_mfp_map* map, uint64_t until,
                                     mzgpu_mfp_op** out) {
  MZ_CHECK_CTX(ctx);
  if (plan == nullptr || out == nullptr) return MZGPU_E_INVALID;
  MfpDevPlan pl;
  MZ_TRY(mfp_build_plan(ctx, plan, map, 0, &pl));
  std::unique_ptr<mzgpu_mfp_op> op;
  MZ_TRY(mfp_op_create(ctx, pl, until, &op));
  *out = op.release();
  return MZGPU_OK;
}

extern "C" void mzgpu_mfp_free(mzgpu_mfp_op* op) { delete op; }

extern "C" int32_t mzgpu_mfp_step(mzgpu_mfp_op* op, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                                  mzgpu_buf* out, mzgpu_buf* errs) {
  if (op == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = op->ctx;
  MZ_CHECK_CTX(ctx);
  const uint32_t irb = op->pl.plan.in_row_bytes;
  ctx->stats.rows_in += n;
  DevMem in;
  const void* d = rows;
  if (mem == MZGPU_MEM_HOST && n) {
    MZ_TRY(in.alloc(ctx, n * irb));
    MZ_TRY(copy_in(ctx, in.p, rows, n * irb, mem));
    d = in.p;
  }
  return mfp_step_dev(op, (const u64*)d, dlen_imm(n), n, upper, out, errs);
}

extern "C" int32_t mzgpu_mfp_step_buf(mzgpu_mfp_op* op, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out,
                                      mzgpu_buf* errs) {
  if (op == nullptr || rows == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(op->ctx);
  if (rows->rb != op->pl.plan.in_row_bytes || rows == out || rows == errs) {
    MZ_SET_ERR(op->ctx, "mfp_step_buf: input rows must be %u bytes wide and not an output buffer",
               op->pl.plan.in_row_bytes);
    return MZGPU_E_INVALID;
  }
  return mfp_step_dev(op, (const u64*)rows->mem.p, buf_dlen(rows), rows->ub, upper, out, errs);
}

extern "C" int32_t mzgpu_mfp_frontier(mzgpu_mfp_op* op, uint64_t* out) {
  if (op == nullptr || out == nullptr) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = op->ctx;
  MZ_CHECK_CTX(ctx);
  MZ_TRY(mfp_poll(op, true));
  MZ_TRY(mfp_flush_pending(op));
  MZ_TRY(mfp_poll(op, true));
  *out = MZGPU_FRONTIER_EMPTY;
  for (auto& kv : op->chain) {
    if (kv.second.slices.empty()) continue;  // (after the poll, every slice left holds rows)
    std::vector<MfpSlices> chunks;
    MfpSlices c;
    c.n = 0;
    for (const MfpSlice& s : kv.second.slices) {
      if (c.n == MZ_MFP_SLICES) {
        chunks.push_back(c);
        c.n = 0;
      }
      c.base[c.n] = s.seg->base();
      c.idx[c.n++] = s.idx;
    }
    chunks.push_back(c);
    MZ_TRY(mz_mfp_min_time(ctx, op->ow, chunks.data(), (u32)chunks.size(), mfp_slices_ub(kv.second.slices),
                           op->dmin()));
    MZ_TRY(copy_out(ctx, out, op->dmin(), 8, MZGPU_MEM_HOST));
    return MZGPU_OK;
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_mfp_stats(mzgpu_mfp_op* op, uint64_t out[3]) {
  if (op == nullptr || out == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(op->ctx);
  MZ_TRY(mfp_poll(op, true));
  MZ_TRY(mfp_flush_pending(op));
  MZ_TRY(mfp_poll(op, true));
  u64 held = 0;
  for (auto& kv : op->chain)
    for (const MfpSlice& s : kv.second.slices) held += mfp_slice_ub(s);
  out[0] = held;
  out[1] = op->chain.size();
  MZ_TRY(copy_out(op->ctx, &out[2], op->touched(), 8, MZGPU_MEM_HOST));
  return MZGPU_OK;
}

// ========================================================== FlatMap
// mzgpu_flat_map_new (include/mzgpu.h): a table function per input row, expanded in pages through the MfpPlan of
// an mzgpu_mfp_op, whose bucket chain holds the future updates.  An activation's rows are copied, their function
// records and inclusive 128-bit counts computed in one pass (mfp.cu: k_fm_count), and the count of function rows
// read back once; every page is one load-balanced expansion (k_fm_expand) followed by steps 2-6 of a mfp step.
typedef unsigned __int128 u128;
struct mzgpu_flat_map_op {
  std::unique_ptr<mzgpu_mfp_op> mfp;
  FlatMapDevPlan pl;
  // the activation in progress
  bool active = false;
  DevMem rows, rec, incl, lb, first_errs;
  u64 n = 0, n_first_errs = 0, upper = 0;
  u128 total = 0, g = 0;  // function rows, and the first not yet expanded
  DevMem d_total;         // total lo, hi, input rows, argument / function errors
};

static int32_t fm_fail(mzgpu_ctx* ctx, int32_t st, const char* what) {
  MZ_SET_ERR(ctx, "flat_map: %s", what);
  return st;
}

extern "C" int32_t mzgpu_flat_map_new(mzgpu_ctx* ctx, const mzgpu_table_func* func, const mzgpu_mfp* plan,
                                      const mzgpu_mfp_map* map, uint64_t until, mzgpu_flat_map_op** out) {
  MZ_CHECK_CTX(ctx);
  if (func == nullptr || plan == nullptr || out == nullptr) return MZGPU_E_INVALID;
  const mzgpu_table_func& tf = *func;
  if (tf.kind < MZGPU_TF_GENERATE_SERIES_INT32 || tf.kind > MZGPU_TF_GUARD_SUBQUERY_SIZE)
    return fm_fail(ctx, MZGPU_E_UNSUPPORTED, "table function outside the fixed-width subset");
  if (tf.with_ordinality > 1) return fm_fail(ctx, MZGPU_E_INVALID, "with_ordinality is 0 or 1");
  if (tf.kind == MZGPU_TF_REPEAT_ROW && tf.with_ordinality)
    return fm_fail(ctx, MZGPU_E_INVALID, "repeat_row WITH ORDINALITY (its diffs may be negative)");
  if (tf.n_consts > MZGPU_MFP_MAX_CONSTS) return fm_fail(ctx, MZGPU_E_INVALID, "argument constants (0..8)");
  const bool series = tf.kind <= MZGPU_TF_GENERATE_SERIES_TIMESTAMP;
  const bool ts = tf.kind == MZGPU_TF_GENERATE_SERIES_TIMESTAMP;
  const uint32_t n_args = ts ? 2 : series ? 3 : 1;
  // the function's columns: the series value, then the ordinal
  const uint32_t n_fn = (series ? 1u : 0u) + tf.with_ordinality;
  FlatMapDevPlan pl;
  memset(&pl, 0, sizeof(pl));
  pl.tf = tf;
  pl.n_args = n_args;
  for (uint32_t a = 0; a < 3; ++a)
    if ((a < n_args) != (tf.n_ops[a] != 0)) return fm_fail(ctx, MZGPU_E_INVALID, "argument count");
  const char* unsupported = nullptr;
  std::string unsupported_msg;
  for (uint32_t a = 0; a < n_args; ++a) {
    const MfpProgram g{MFP_MAP, a, tf.ops[a], tf.n_ops[a], tf.consts, tf.n_consts, pl.iv_us, nullptr, 0, 0};
    MfpTy t;
    uint32_t support;
    MZ_TRY(validate_mfp_program(ctx, plan->in_row_bytes, g, &t, &support, &unsupported));
    if (unsupported && unsupported_msg.empty()) unsupported_msg = ctx->last_error;
    const bool ok = ts ? t == MFP_TS
                       : tf.kind == MZGPU_TF_GENERATE_SERIES_INT32 ? t == MFP_INT32 : t == MFP_INT32 || t == MFP_INT64;
    if (!ok) {
      MZ_SET_ERR(ctx, "flat_map: argument %u has the wrong type", a);
      return MZGPU_E_INVALID;
    }
  }
  if (ts) {
    const mzgpu_having_const& k = tf.step_iv;
    const int32_t days = (int32_t)(uint32_t)k.hi, months = (int32_t)(uint32_t)(k.hi >> 32);
    const __int128 us = (__int128)days * 86400000000ll + (__int128)(int64_t)k.lo;
    if (months != 0 && !unsupported) {
      MZ_SET_ERR(ctx, "flat_map: a timestamp series step with months");
      unsupported = "months";
      unsupported_msg = ctx->last_error;
    } else if ((us < (__int128)INT64_MIN || us > (__int128)INT64_MAX) && !unsupported) {
      MZ_SET_ERR(ctx, "flat_map: a timestamp series step beyond i64 microseconds");
      unsupported = "step";
      unsupported_msg = ctx->last_error;
    } else {
      pl.step_us = (i64)us;
    }
  }
  const int32_t st = mfp_build_plan(ctx, plan, map, n_fn, &pl.mfp);
  if (st == MZGPU_E_INVALID) return st;
  if (unsupported) {
    ctx->last_error = unsupported_msg;
    return MZGPU_E_UNSUPPORTED;
  }
  MZ_TRY(st);
  auto op = std::unique_ptr<mzgpu_flat_map_op>(new mzgpu_flat_map_op());
  MZ_TRY(mfp_op_create(ctx, pl.mfp, until, &op->mfp));
  op->pl = pl;
  MZ_TRY(op->d_total.alloc(ctx, 4 * 8));
  *out = op.release();
  return MZGPU_OK;
}

extern "C" void mzgpu_flat_map_free(mzgpu_flat_map_op* op) { delete op; }

// One page: the next `fuel` function rows of the activation through the MfpPlan (the first page also carries the
// argument and function errors), then steps 2-6 of a mfp step.
static int32_t fm_page(mzgpu_flat_map_op* op, uint64_t fuel, mzgpu_buf* out, mzgpu_buf* errs, int32_t* done) {
  mzgpu_mfp_op* m = op->mfp.get();
  mzgpu_ctx* ctx = m->ctx;
  const u128 left = op->total - op->g;
  const u64 page = left < (u128)fuel ? (u64)left : fuel;
  MZ_TRY(mfp_step_begin(m));
  std::shared_ptr<MfpSeg> ready, held;
  MZ_TRY(mfp_segments(m, 2 * page, &ready, &held));
  const u64 err_ub = op->n_first_errs + page;
  DevMem err_rows;
  Lazy4 err_len;
  if (err_ub > 0) {
    MZ_TRY(err_rows.alloc(ctx, err_ub * 32));
    MZ_TRY(err_len.make_pending(ctx));
    const u64 k = op->n_first_errs;
    if (k) {
      MZ_TRY(copy_out(ctx, err_len.dptr(), (const u64*)op->d_total.p + 3, 8, MZGPU_MEM_DEVICE));
      MZ_TRY(copy_out(ctx, err_rows.p, op->first_errs.p, k * 32, MZGPU_MEM_DEVICE));
    } else {
      MZ_CUDA(ctx, cudaMemsetAsync(err_len.dptr(), 0, 8, ctx->stream));
    }
  }
  if (page > 0)
    MZ_TRY(mz_fm_expand(ctx, op->pl, (const u64*)op->rows.p, (const FmRec*)op->rec.p, (const ulonglong2*)op->incl.p,
                        op->n, op->g, page, op->upper, m->until, ready->base(), held->base(), (u64*)err_rows.p,
                        err_len.dptr()));
  if (err_ub > 0) err_len.mark_written();
  MZ_TRY(mfp_step_end(m, ready, held, (const u64*)err_rows.p, err_ub > 0 ? dlen_of(err_len, 0) : dlen_imm(0), err_ub,
                      op->upper, out, errs));
  op->g += page;
  op->n_first_errs = 0;
  op->first_errs.release();
  if (op->g == op->total) {
    op->active = false;
    op->rows.release();
    op->rec.release();
    op->incl.release();
    op->lb.release();
  }
  *done = op->active ? 0 : 1;
  return MZGPU_OK;
}

static int32_t fm_step_dev(mzgpu_flat_map_op* op, const void* d_rows, int32_t mem, DLen n, u64 n_ub, uint64_t upper,
                           uint64_t fuel, mzgpu_buf* out, mzgpu_buf* errs, int32_t* done) {
  mzgpu_mfp_op* m = op->mfp.get();
  mzgpu_ctx* ctx = m->ctx;
  if (done == nullptr || fuel == 0) return fm_fail(ctx, MZGPU_E_INVALID, "step needs fuel > 0 and a done flag");
  if (op->active) return fm_fail(ctx, MZGPU_E_FRONTIER, "step while an activation is unfinished (call work)");
  MZ_TRY(mfp_step_check(m, upper, out, errs));
  const u64 irb = op->pl.mfp.plan.in_row_bytes;
  op->total = op->g = 0;
  op->n = op->n_first_errs = 0;
  if (n_ub > 0) {
    // the rows are copied: the caller's buffer is free once the step returns
    MZ_TRY(op->rows.alloc(ctx, n_ub * irb));
    MZ_TRY(copy_in(ctx, op->rows.p, d_rows, n_ub * irb, mem));
    const u64 n_tiles = (n_ub + MZ_FM_TILE - 1) / MZ_FM_TILE;
    MZ_TRY(op->rec.alloc(ctx, n_ub * sizeof(FmRec)));
    MZ_TRY(op->incl.alloc(ctx, n_ub * 16));
    MZ_TRY(op->lb.alloc(ctx, (n_tiles * 5 + 1) * 8));
    MZ_TRY(op->first_errs.alloc(ctx, n_ub * 32));
    u64* tot = (u64*)op->d_total.p;
    MZ_CUDA(ctx, cudaMemsetAsync(tot, 0, 4 * 8, ctx->stream));
    MZ_TRY(mz_fm_count(ctx, op->pl, (const u64*)op->rows.p, n, n_ub, (FmRec*)op->rec.p, (ulonglong2*)op->incl.p,
                       (u64*)op->lb.p, tot, (u64*)op->first_errs.p, tot + 3));
    u64 h[4];
    MZ_TRY(copy_out(ctx, h, tot, sizeof(h), MZGPU_MEM_HOST));  // the activation's one wait
    op->total = ((u128)h[1] << 64) | h[0];
    op->n = h[2];
    op->n_first_errs = h[3];
  }
  op->active = true;
  op->upper = upper;
  return fm_page(op, fuel, out, errs, done);
}

extern "C" int32_t mzgpu_flat_map_step(mzgpu_flat_map_op* op, const void* rows, uint64_t n, int32_t mem,
                                       uint64_t upper, uint64_t fuel, mzgpu_buf* out, mzgpu_buf* errs, int32_t* done) {
  if (op == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(op->mfp->ctx);
  op->mfp->ctx->stats.rows_in += n;
  return fm_step_dev(op, rows, mem, dlen_imm(n), n, upper, fuel, out, errs, done);
}

extern "C" int32_t mzgpu_flat_map_step_buf(mzgpu_flat_map_op* op, mzgpu_buf* rows, uint64_t upper, uint64_t fuel,
                                           mzgpu_buf* out, mzgpu_buf* errs, int32_t* done) {
  if (op == nullptr || rows == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(op->mfp->ctx);
  if (rows->rb != op->pl.mfp.plan.in_row_bytes || rows == out || rows == errs)
    return fm_fail(op->mfp->ctx, MZGPU_E_INVALID, "step_buf: input rows of the plan's width, not an output buffer");
  return fm_step_dev(op, rows->mem.p, MZGPU_MEM_DEVICE, buf_dlen(rows), rows->ub, upper, fuel, out, errs, done);
}

extern "C" int32_t mzgpu_flat_map_work(mzgpu_flat_map_op* op, uint64_t fuel, mzgpu_buf* out, mzgpu_buf* errs,
                                       int32_t* done) {
  if (op == nullptr || done == nullptr) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = op->mfp->ctx;
  MZ_CHECK_CTX(ctx);
  if (fuel == 0) return fm_fail(ctx, MZGPU_E_INVALID, "work needs fuel > 0");
  if (!op->active) {
    *done = 1;
    return MZGPU_OK;
  }
  MZ_TRY(mfp_step_check(op->mfp.get(), op->upper, out, errs));
  return fm_page(op, fuel, out, errs, done);
}

extern "C" int32_t mzgpu_flat_map_frontier(mzgpu_flat_map_op* op, uint64_t* out) {
  if (op == nullptr || out == nullptr) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = op->mfp->ctx;
  MZ_CHECK_CTX(ctx);
  u64 t = MZGPU_FRONTIER_EMPTY;
  MZ_TRY(mzgpu_mfp_frontier(op->mfp.get(), &t));
  if (op->active && op->n > 0) {
    u64* dmin = op->mfp->dmin();
    MZ_CUDA(ctx, cudaMemsetAsync(dmin, 0xff, 8, ctx->stream));
    MZ_TRY(mz_fm_min_time(ctx, (int)op->pl.mfp.plan.in_row_bytes, (const u64*)op->rows.p,
                          (const ulonglong2*)op->incl.p, op->n, op->g, dmin));
    u64 pend;
    MZ_TRY(copy_out(ctx, &pend, dmin, 8, MZGPU_MEM_HOST));
    if (pend != ~0ull && (t == MZGPU_FRONTIER_EMPTY || pend < t)) t = pend;
  }
  *out = t;
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_flat_map_stats(mzgpu_flat_map_op* op, uint64_t out[4]) {
  if (op == nullptr || out == nullptr) return MZGPU_E_INVALID;
  MZ_TRY(mzgpu_mfp_stats(op->mfp.get(), out));
  const u128 left = op->active ? op->total - op->g : 0;
  out[3] = left > (u128)~0ull ? ~0ull : (u64)left;
  return MZGPU_OK;
}

// ============================================================ index peeks
// mzgpu_peek_many: gather every request's pairs (full scans and literal lookups) into one R40 buffer of rows
// (slot, key, val, as_of, diff), consolidate it once, evaluate each request's plan per pair, consolidate the
// finishing rows once (their word order is the finishing order), cut and project per request, and read the k
// results back with one wait.
static_assert(MZ_PEEK_K == MZGPU_PEEK_MANY_MAX, "one request slot per request of a call");
struct mzgpu_peek_plan {
  mzgpu_ctx* ctx;
  uint32_t out_rb;
  DevMem dev;  // PeekDevPlan
};

// a finishing field: a bit-field of an output word (VAL2 only of 40-byte output)
static int32_t peek_field_check(mzgpu_ctx* ctx, const char* what, uint32_t i, const mzgpu_field& f, uint32_t out_rb,
                                bool uses_dst) {
  const uint32_t max_src = out_rb == 40 ? MZGPU_SRC_VAL2 : MZGPU_SRC_VAL1;
  if (f.src > max_src || f.bits < 1 || f.bits > 64 || f.shift > 63 || (uint32_t)f.shift + f.bits > 64 ||
      (uses_dst && f.dst_shift >= 64)) {
    MZ_SET_ERR(ctx, "peek plan: %s %u is not a bit-field of the %u-byte output row", what, i, out_rb);
    return MZGPU_E_INVALID;
  }
  return MZGPU_OK;
}

static int32_t peek_finishing(mzgpu_ctx* ctx, const mzgpu_finishing* fin, uint32_t out_rb, PeekFin* F) {
  F->out_words = out_rb / 8 - 2;
  F->offset = 0;
  F->end = ~0ull;
  F->identity = 1;
  if (fin == nullptr) return MZGPU_OK;
  if (fin->n_order > MZGPU_MAX_ORDER_LANES) {
    MZ_SET_ERR(ctx, "peek plan: %u order lanes (0..%d)", fin->n_order, MZGPU_MAX_ORDER_LANES);
    return MZGPU_E_INVALID;
  }
  int unsupported = -1;
  for (uint32_t j = 0; j < fin->n_order; ++j) {
    const mzgpu_order_lane& L = fin->order[j];
    if ((L.flags & ~(uint32_t)MZGPU_ORDER_F64) != 0) {
      MZ_SET_ERR(ctx, "peek plan: order lane %u: unknown flag bits", j);
      return MZGPU_E_INVALID;
    }
    MZ_TRY(peek_field_check(ctx, "order lane", j, L.field, out_rb, false));
    if ((L.flags & MZGPU_ORDER_F64) != 0 && unsupported < 0) unsupported = (int)j;
    F->f[j] = L.field;
    F->sign_extend[j] = L.sign_extend != 0;
    F->xm[j] = (L.sign_extend ? 1ull << 63 : 0) ^ (L.descending ? ~0ull : 0);
  }
  for (uint32_t w = 0; w < 3; ++w) {
    if (fin->n_project[w] > MZGPU_MAX_FIELDS || (w >= F->out_words && fin->n_project[w] != 0)) {
      MZ_SET_ERR(ctx, "peek plan: %u projection fields for word %u of a %u-byte row", fin->n_project[w], w, out_rb);
      return MZGPU_E_INVALID;
    }
    for (uint32_t i = 0; i < fin->n_project[w]; ++i)
      MZ_TRY(peek_field_check(ctx, "projection field", i, fin->project[w][i], out_rb, true));
    F->n_project[w] = fin->n_project[w];
    for (uint32_t i = 0; i < fin->n_project[w]; ++i) F->project[w][i] = fin->project[w][i];
    if (fin->n_project[w] != 0) F->identity = 0;
  }
  if (unsupported >= 0) {
    MZ_SET_ERR(ctx, "peek plan: order lane %d: float64 order columns are not supported (OrderedFloat ties -0.0 with "
                    "+0.0 and NaN payloads)", unsupported);
    return MZGPU_E_UNSUPPORTED;
  }
  if (fin->limit < 0) {
    MZ_SET_ERR(ctx, "peek plan: negative limit %lld", (long long)fin->limit);
    return MZGPU_E_UNSUPPORTED;
  }
  F->n_order = fin->n_order;
  F->offset = fin->offset;
  if (fin->limit != MZGPU_TOPK_NO_LIMIT) {
    const u64 lim = (u64)fin->limit;
    F->end = fin->offset > ~0ull - lim ? ~0ull : fin->offset + lim;
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_peek_plan_new(mzgpu_ctx* ctx, const mzgpu_mfp* plan, const mzgpu_mfp_map* map,
                                       const mzgpu_finishing* fin, mzgpu_peek_plan** out) {
  MZ_CHECK_CTX(ctx);
  if (plan == nullptr || out == nullptr) return MZGPU_E_INVALID;
  if (plan->in_row_bytes != 32) {
    MZ_SET_ERR(ctx, "peek plan: the input is the trace's (key, val), in_row_bytes 32, not %u", plan->in_row_bytes);
    return MZGPU_E_INVALID;
  }
  if (plan->n_temporal != 0) {
    MZ_SET_ERR(ctx, "peek plan: %u temporal predicates (a peek's plan is a SafeMfpPlan)", plan->n_temporal);
    return MZGPU_E_INVALID;
  }
  std::unique_ptr<PeekDevPlan> pd(new PeekDevPlan());
  memset(pd.get(), 0, sizeof(PeekDevPlan));
  MZ_TRY(mfp_build_plan(ctx, plan, map, 0, &pd->mfp));
  MZ_TRY(peek_finishing(ctx, fin, plan->out_row_bytes, &pd->fin));
  auto p = std::unique_ptr<mzgpu_peek_plan>(new mzgpu_peek_plan());
  p->ctx = ctx;
  p->out_rb = plan->out_row_bytes;
  MZ_TRY(p->dev.alloc(ctx, sizeof(PeekDevPlan)));
  MZ_TRY(copy_in(ctx, p->dev.p, pd.get(), sizeof(PeekDevPlan), MZGPU_MEM_HOST));
  *out = p.release();
  return MZGPU_OK;
}
extern "C" void mzgpu_peek_plan_free(mzgpu_peek_plan* p) { delete p; }

// rows of the readable batches (upper bounds for batches still in flight)
static u64 peek_rows_ub(const std::vector<mzgpu_batch*>& bs) {
  u64 n = 0;
  for (auto* b : bs) n += b->st.known ? b->st.v[0] : b->len_ub;
  return n;
}

// The literal requests' keys, deduplicated per request, looked up by the half-join probe: the stream rows
// (key, slot, as_of, +1) under an identity MfpPlan that writes (slot, key, val) appends R40 rows to `g`.
static int32_t peek_literals(mzgpu_ctx* ctx, const std::vector<mzgpu_batch*>& okb, const mzgpu_peek_req* reqs,
                             const PeekLitSegs& segs, mzgpu_buf* g) {
  const u64 n = segs.start[segs.n];
  DevMem keys, rows, cons;
  MZ_TRY(keys.alloc(ctx, n * 8));
  for (u32 s = 0; s < segs.n; ++s) {
    const mzgpu_peek_req& r = reqs[segs.slot[s]];
    MZ_TRY(copy_in(ctx, keys.as<u64>() + segs.start[s], r.literals, r.n_literals * 8, r.literals_mem));
  }
  MZ_TRY(rows.alloc(ctx, n * 32));
  MZ_TRY(mz_peek_lits(ctx, keys.as<u64>(), segs, rows.as<u64>()));
  u64 ccap = 0;
  Lazy4 clen;
  MZ_TRY(consolidate_dev(ctx, 32, rows.p, dlen_imm(n), n, &cons, &ccap, &clen));
  const DLen sn = dlen_of(clen, 0);
  const u64 s_ub = clen.known ? clen.v[0] : std::min(ccap, n);
  MZ_TRY(mz_peek_unit(ctx, cons.as<u64>(), sn, s_ub));
  mzgpu_mfp idp;
  memset(&idp, 0, sizeof(idp));
  idp.in_row_bytes = idp.out_row_bytes = 40;
  idp.n_fields[0] = idp.n_fields[1] = idp.n_fields[2] = 1;
  idp.fields[0][0] = mzgpu_field{MZGPU_SRC_VAL1, 0, 64, 0};
  idp.fields[1][0] = mzgpu_field{MZGPU_SRC_KEY, 0, 64, 0};
  idp.fields[2][0] = mzgpu_field{MZGPU_SRC_VAL2, 0, 64, 0};
  std::unique_ptr<mzgpu_join_closure> idc(new mzgpu_join_closure());
  idc->ctx = ctx;
  MZ_TRY(mfp_build_plan(ctx, &idp, nullptr, 0, &idc->pl));
  MZ_TRY(idc->dev.alloc(ctx, sizeof(MfpDevPlan)));
  MZ_TRY(copy_in(ctx, idc->dev.p, &idc->pl, sizeof(MfpDevPlan), MZGPU_MEM_HOST));
  std::unique_ptr<TraceView> tv(new TraceView());
  ProbePlan p;
  MZ_TRY(probe_plan(ctx, okb, MZ_PROBE_HALF_LE, nullptr, 0, false, MZ_BOUND_MAX_ROWS * 32 / (40 + 32), tv.get(), &p,
                    idc.get()));
  ErrSink es;  // the identity plan raises no error
  return probe_run(ctx, p, cons.as<u64>(), sn, s_ub, ProbeOut::APPEND, g, nullptr, &es);
}

extern "C" int32_t mzgpu_peek_many(mzgpu_ctx* ctx, mzgpu_spine* ok, mzgpu_spine* errs, uint32_t k,
                                   const mzgpu_peek_req* reqs, mzgpu_buf* const* outs, mzgpu_peek_result* results) {
  MZ_CHECK_CTX(ctx);
  if (ok == nullptr || reqs == nullptr || outs == nullptr || results == nullptr || k == 0 || k > MZGPU_PEEK_MANY_MAX) {
    MZ_SET_ERR(ctx, "peek: bad arguments (k = %u, 1..%d)", k, MZGPU_PEEK_MANY_MAX);
    return MZGPU_E_INVALID;
  }
  if (ok->ctx != ctx || ok->rb != 32 || (errs != nullptr && (errs->ctx != ctx || errs->rb != 32))) {
    MZ_SET_ERR(ctx, "peek: the ok and error traces are R32 arrangements of this context");
    return MZGPU_E_INVALID;
  }
  for (uint32_t i = 0; i < k; ++i) {
    const mzgpu_peek_req& r = reqs[i];
    if (r.plan == nullptr || r.plan->ctx != ctx || outs[i] == nullptr || outs[i]->ctx != ctx ||
        outs[i]->rb != r.plan->out_rb || (r.literals == nullptr && r.n_literals != 0) ||
        (r.literals_mem != MZGPU_MEM_HOST && r.literals_mem != MZGPU_MEM_DEVICE)) {
      MZ_SET_ERR(ctx, "peek: request %u: bad plan, output buffer or literal list", i);
      return MZGPU_E_INVALID;
    }
  }
  // the frontier checks of seek_fulfillment, on the host
  const u64 since = std::max(ok->since, errs != nullptr ? errs->since : 0);
  auto not_ready = [](const mzgpu_spine* s, u64 t) { return s->upper != MZGPU_FRONTIER_EMPTY && s->upper <= t; };
  PeekReqs rq;
  memset(&rq, 0, sizeof(rq));
  rq.k = k;
  PeekScanJobs ok_jobs, err_jobs;
  memset(&ok_jobs, 0, sizeof(ok_jobs));
  memset(&err_jobs, 0, sizeof(err_jobs));
  PeekLitSegs segs;
  memset(&segs, 0, sizeof(segs));
  bool any = false;
  u64 n_scan_reqs = 0;  // full-scan requests (each slot of the ok trace's scans is shared by the requests at its as_of)
  for (uint32_t i = 0; i < k; ++i) {
    const mzgpu_peek_req& r = reqs[i];
    mzgpu_peek_result& res = results[i];
    memset(&res, 0, sizeof(res));
    rq.err_slot[i] = -1;
    if (not_ready(ok, r.as_of) || (errs != nullptr && not_ready(errs, r.as_of))) {
      res.status = MZGPU_PEEK_NOT_READY;
      continue;
    }
    if (since > r.as_of) {
      res.status = MZGPU_PEEK_ERROR;
      res.err_kind = MZGPU_PEEK_ERR_SINCE;
      res.detail[0] = since;
      res.detail[1] = r.as_of;
      continue;
    }
    any = true;
    rq.pl[i] = r.plan->dev.as<PeekDevPlan>();
    rq.as_of[i] = r.as_of;
    if (errs != nullptr) {  // one error-trace scan per distinct as_of (its slot is numbered below)
      uint32_t j = 0;
      while (j < err_jobs.n && err_jobs.as_of[j] != r.as_of) ++j;
      if (j == err_jobs.n) err_jobs.as_of[err_jobs.n++] = r.as_of;
      rq.err_slot[i] = (int)j;
    }
    if (r.literals == nullptr) {  // one ok-trace scan per distinct as_of, shared by its requests
      uint32_t j = 0;
      while (j < ok_jobs.n && ok_jobs.as_of[j] != r.as_of) ++j;
      if (j == ok_jobs.n) {
        ok_jobs.slot[j] = k + j;
        ok_jobs.as_of[ok_jobs.n++] = r.as_of;
      }
      rq.reqs[k + j] |= 1ull << i;
      n_scan_reqs++;
    } else if (r.n_literals != 0) {
      segs.slot[segs.n] = i;
      segs.as_of[segs.n] = r.as_of;
      segs.start[segs.n + 1] = segs.start[segs.n] + r.n_literals;
      segs.n++;
      rq.reqs[i] = 1ull << i;
    }
  }
  rq.err_base = k + ok_jobs.n;
  for (uint32_t j = 0; j < err_jobs.n; ++j) err_jobs.slot[j] = rq.err_base + j;
  for (uint32_t i = 0; i < k; ++i)
    if (rq.err_slot[i] >= 0) rq.err_slot[i] += (int)rq.err_base;
  if (!any) return MZGPU_OK;

  // 1. gather
  std::vector<mzgpu_batch*> okb, errb;
  spine_readable(ok, okb);
  if (errs != nullptr) spine_readable(errs, errb);
  std::unique_ptr<TraceView> tv_ok(new TraceView()), tv_err(new TraceView());
  MZ_TRY(trace_view(ctx, okb, tv_ok.get()));
  if (errs != nullptr) MZ_TRY(trace_view(ctx, errb, tv_err.get()));
  mzgpu_buf g;
  g.ctx = ctx;
  g.rb = 40;
  g.len.set(ctx, 0);
  const u64 ok_rows = peek_rows_ub(okb);
  const u64 scan_ub = ok_rows * ok_jobs.n + peek_rows_ub(errb) * err_jobs.n;
  if (scan_ub != 0) {
    MZ_TRY(buf_reserve(&g, scan_ub, false));
    Append a;
    MZ_TRY(buf_begin_append(&g, &a));  // (g is empty: the scans count from 0)
    MZ_CUDA(ctx, cudaMemsetAsync(a.out_len, 0, 8, ctx->stream));
    MZ_TRY(mz_peek_scan(ctx, *tv_ok, ok_jobs, g.mem.as<u64>(), g.cap, a.out_len));
    if (errs != nullptr) MZ_TRY(mz_peek_scan(ctx, *tv_err, err_jobs, g.mem.as<u64>(), g.cap, a.out_len));
    buf_end_append(&g, a, scan_ub);
  }
  if (segs.n != 0) MZ_TRY(peek_literals(ctx, okb, reqs, segs, &g));

  // 2. accumulate, 3. evaluate, 4. finish
  std::vector<PeekDevResult> hres(k);
  memset(hres.data(), 0, k * sizeof(PeekDevResult));
  DevMem pairs, fail, fin, fcons, stage, dres;
  if (g.ub != 0) {
    u64 pcap = 0;
    Lazy4 plen;
    MZ_TRY(consolidate_dev(ctx, 40, g.mem.p, buf_dlen(&g), g.ub, &pairs, &pcap, &plen));
    const DLen pn = dlen_of(plen, 0);
    const u64 p_ub = plen.known ? plen.v[0] : std::min(pcap, g.ub);
    const u64 n_slots = rq.err_base + err_jobs.n;  // fail[request] and fail[error-trace slot]
    MZ_TRY(fail.alloc(ctx, n_slots * 8));
    MZ_CUDA(ctx, cudaMemsetAsync(fail.p, 0xff, n_slots * 8, ctx->stream));
    // finishing rows: a literal request's pair gives at most one, a scanned pair one per request at its as_of
    u64 share = 1;
    for (uint32_t j = 0; j < ok_jobs.n; ++j) share = std::max<u64>(share, __builtin_popcountll(rq.reqs[k + j]));
    const u64 fin_ub = std::min(p_ub * share, n_scan_reqs * std::min(ok_rows, p_ub) + p_ub);
    MZ_TRY(fin.alloc(ctx, std::max<u64>(fin_ub, 1) * 72));
    Lazy4 flen;
    MZ_TRY(flen.make_pending(ctx));
    MZ_CUDA(ctx, cudaMemsetAsync(flen.dptr(), 0, 8, ctx->stream));
    MZ_TRY(mz_peek_eval(ctx, pairs.as<u64>(), pn, p_ub, fin_ub, rq, fin.as<u64>(), flen.dptr(), fail.as<u64>()));
    flen.mark_written();
    u64 fcap = 0;
    Lazy4 fclen;
    DLen fn = dlen_imm(0);
    u64 f_ub = 0;
    if (fin_ub != 0) {
      MZ_TRY(consolidate_dev(ctx, 72, fin.p, dlen_of(flen, 0), fin_ub, &fcons, &fcap, &fclen));
      fn = dlen_of(fclen, 0);
      f_ub = fclen.known ? fclen.v[0] : std::min(fcap, fin_ub);
    }
    MZ_TRY(stage.alloc(ctx, std::max<u64>(f_ub, 1) * 40));
    MZ_TRY(dres.alloc(ctx, k * sizeof(PeekDevResult)));
    MZ_CUDA(ctx, cudaMemsetAsync(dres.p, 0, k * sizeof(PeekDevResult), ctx->stream));
    MZ_TRY(mz_peek_finish(ctx, rq, pairs.as<u64>(), fail.as<u64>(), fcons.as<u64>(), fn, stage.as<u64>(),
                          dres.as<PeekDevResult>()));
    MZ_TRY(copy_out(ctx, hres.data(), dres.p, k * sizeof(PeekDevResult), MZGPU_MEM_HOST));  // the one wait
  }
  for (uint32_t i = 0; i < k; ++i) {
    if (rq.pl[i] == nullptr) continue;
    const PeekDevResult& d = hres[i];
    mzgpu_peek_result& res = results[i];
    if (d.kind != 0) {
      res.status = MZGPU_PEEK_ERROR;
      res.err_kind = (int32_t)d.kind;
      for (int w = 0; w < 4; ++w) res.detail[w] = d.d[w];
    } else if (reqs[i].max_rows != 0 && d.n_rows > reqs[i].max_rows) {
      res.status = MZGPU_PEEK_ERROR;
      res.err_kind = MZGPU_PEEK_ERR_TOO_LARGE;
      res.detail[0] = d.n_rows;
    } else {
      res.status = MZGPU_PEEK_ROWS;
      res.n_rows = d.n_rows;
      if (d.n_rows != 0)
        MZ_TRY(buf_append_dev(outs[i], (const char*)stage.p + d.lo * 40, dlen_imm(d.n_rows), d.n_rows));
      ctx->stats.rows_out += d.n_rows;
    }
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_peek(mzgpu_ctx* ctx, mzgpu_spine* ok, mzgpu_spine* errs, const mzgpu_peek_req* req,
                              mzgpu_buf* out, mzgpu_peek_result* result) {
  return mzgpu_peek_many(ctx, ok, errs, 1, req, &out, result);
}
