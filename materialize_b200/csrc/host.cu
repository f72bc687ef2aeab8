// host.cu — the C ABI of libmzgpu (include/mzgpu.h): contexts, row buffers,
// batcher, batches, the fueled spine, join_core / half_join / reduce operator
// state, and the NCCL exchange.  Host-side bookkeeping only; every per-row
// operation is a CUDA kernel from the sibling .cu files.  There is no CPU
// fallback: without a CUDA device every entry point fails with MZGPU_E_CUDA.
#include <dlfcn.h>

#include <algorithm>
#include <cstring>
#include <deque>
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

// arrangement rows: every sorted-batch width but the reduce's 64-byte output rows, i.e. R32 and the
// accumulable rows of every lane class (RACC = class 1)
static bool arrangement_row_bytes(uint32_t rb) { return rb != 64 && BatchWidths::has((int)rb); }
// buffer rows: every RowT width, and the wide output rows of the lanes reduce (they have no RowT)
static bool valid_row_bytes(uint32_t rb) { return RowWidths::has((int)rb) || rb == 96 || rb == 144 || rb == 240; }

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
// rows (device, count possibly device resident) -> consolidated rows; the fused
// kernel for small / medium inputs, the multi-kernel path beyond.
static int32_t consolidate_dev(mzgpu_ctx* ctx, int rb, const void* d_in, DLen n, u64 n_ub, DevMem* out,
                               u64* out_cap, Lazy4* out_len) {
  if (n.p != nullptr && !mz_use_fused(false, n_ub)) {
    // bound too loose to size buffers by: read the count back
    MZ_TRY(mz_resolve_counters(ctx));
    n = dlen_imm(ctx->h_cnt[n.p - ctx->d_cnt]);  // the block is part of the arena mirror
    n_ub = n.imm;
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
  const int tw = b->rb == 32 ? 2 : 1;
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

// ================================================================ join_core
struct mzgpu_join {
  mzgpu_ctx* ctx;
  mzgpu_spine *t1, *t2;
  bool has_closure;
  mzgpu_closure closure;
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

extern "C" int32_t mzgpu_join_new(mzgpu_ctx* ctx, mzgpu_spine* trace1, mzgpu_spine* trace2,
                                  const mzgpu_closure* closure, mzgpu_join** out) {
  MZ_CHECK_CTX(ctx);
  if (trace1 == nullptr || trace2 == nullptr || out == nullptr || trace1->rb != 32 || trace2->rb != 32)
    return MZGPU_E_INVALID;
  MZ_TRY(validate_closure(ctx, closure));
  mzgpu_join* j = new mzgpu_join();
  j->ctx = ctx;
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
extern "C" int32_t mzgpu_join_core_work_until(mzgpu_join* j, uint64_t fuel_rows, uint64_t deadline_ns,
                                              mzgpu_buf* out, int32_t* done) {
  if (j == nullptr || out == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(j->ctx);
  const uint32_t out_rb = j->has_closure ? 32 : 40;
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
    TraceView tv;
    int32_t st = MZGPU_OK;
    for (auto* b : w.others)
      if (st == MZGPU_OK) st = batch_resolve(b);
    if (st == MZGPU_OK) st = batch_ready(w.batch);
    if (st == MZGPU_OK) st = batch_resolve(w.batch);
    if (st == MZGPU_OK) st = trace_view(j->ctx, w.others, &tv);
    DevMem res, cons;
    u64 n_res = 0, ccap = 0;
    Lazy4 clen;
    // this slice: rows [w.pos, w.pos + n_probe) of the work item's batch
    const u64 n_total = st == MZGPU_OK ? w.batch->st.v[0] : 0;
    // a caller that gave no deadline and has fuel left for more than one slice is not asking to be
    // yielded to: it gets slices as large as its fuel allows (up to 16M rows), which take the bulk
    // sort for the slice's output instead of ten 1M-row fused launches (BASELINE config 2)
    u64 slice = MZ_JOIN_SLICE_ROWS;
    if (deadline_ns == 0) slice = std::max<u64>(slice, std::min<u64>(fuel_rows - produced, 16ull << 20));
    const u64 n_probe = std::min<u64>(n_total - std::min(n_total, w.pos), slice);
    const u64* d_probe = w.batch->rows.as<u64>() + w.pos * 4;
    if (st == MZGPU_OK && n_probe > 0) {
      ProbeParams pp;
      memset(&pp, 0, sizeof(pp));
      pp.mode = MZ_PROBE_JOIN;
      pp.meet = w.cap;
      pp.has_closure = j->has_closure ? 1 : 0;
      pp.swap_vals = w.side == 1 ? 1 : 0;
      pp.closure = j->closure;
      // Bounded fan-out: one pass into a buffer of n x (sum of the longest key runs) rows -- the
      // probe walks the trace once instead of twice (count, write) and the only read-back is the
      // result count that the fuel accounting needs anyway.
      u64 fan = 0;
      bool exact = true;
      st = trace_fanout(w.others, &fan, &exact);
      const bool bounded = st == MZGPU_OK && exact && fan > 0 &&
                           n_probe <= MZ_BULK_BOUND_BYTES / (fan * out_rb) && mz_probe_tiles(n_probe, tv.n_batches) <= MZ_LB_TILES;
      if (st == MZGPU_OK && bounded) {
        Lazy4 rlen;
        const u64 bound = n_probe * fan;
        st = res.alloc(j->ctx, bound * out_rb);
        if (st == MZGPU_OK) st = rlen.make_pending(j->ctx);
        if (st == MZGPU_OK) {
          st = mz_probe_async(j->ctx, d_probe, dlen_imm(n_probe), n_probe, tv, pp, res.as<u64>(), dlen_imm(0), bound,
                              rlen.dptr());
          rlen.mark_written();
        }
        if (st == MZGPU_OK) st = rlen.resolve();
        if (st == MZGPU_OK) n_res = rlen.v[0];
      } else if (st == MZGPU_OK) {
        st = mz_probe(j->ctx, d_probe, n_probe, tv, pp, &res, &n_res);
      }
    }
    // Work::process consolidates each work item's output buffer before sending
    if (st == MZGPU_OK && n_res)
      st = consolidate_dev(j->ctx, out_rb, res.p, dlen_imm(n_res), n_res, &cons, &ccap, &clen);
    if (st == MZGPU_OK && n_res) st = clen.resolve();
    const u64 n_cons = n_res ? clen.v[0] : 0;
    if (st == MZGPU_OK && n_cons) st = buf_append_dev(out, cons.p, dlen_imm(n_cons), n_cons);
    if (st != MZGPU_OK) return st;
    w.pos += n_probe;
    if (w.pos >= n_total) {
      j->release_work(w);
      j->todo.pop_front();
    }
    produced += n_cons;
    j->ctx->stats.rows_out += n_cons;
  }
  if (done) *done = j->todo.empty() ? 1 : 0;
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_join_core_work(mzgpu_join* j, uint64_t fuel_rows, mzgpu_buf* out, int32_t* done) {
  return mzgpu_join_core_work_until(j, fuel_rows, 0, out, done);
}

// ================================================================ half_join
// Bounded probes run in one pass with no host round trip: the capacity
// n_ub x (sum over batches of the longest key run) cannot be exceeded.  Beyond
// MZ_BOUND_MAX_ROWS (heavy skew) the exact two-pass form (count, read back,
// write) is used.
#define MZ_BOUND_MAX_ROWS (48ull << 20)

static int32_t half_join_dev(mzgpu_ctx* ctx, const u64* d_stream, DLen n, u64 n_ub, mzgpu_spine* trace,
                             int32_t cmp_mode, const mzgpu_closure* closure, int32_t consolidate_output,
                             mzgpu_buf* out) {
  if (n_ub == 0) return MZGPU_OK;
  std::vector<mzgpu_batch*> all;
  spine_readable(trace, all);
  u64 fan = 0;
  bool exact = true;
  MZ_TRY(trace_fanout(all, &fan, &exact));
  TraceView tv;
  MZ_TRY(trace_view(ctx, all, &tv));
  if (tv.n_batches == 0) return MZGPU_OK;
  ProbeParams pp;
  memset(&pp, 0, sizeof(pp));
  pp.mode = cmp_mode == MZGPU_HALFJOIN_LE ? MZ_PROBE_HALF_LE : MZ_PROBE_HALF_LT;
  pp.has_closure = 1;
  if (closure) {
    pp.closure = *closure;
  } else {
    // identity on (key, val2): the lookup value replaces the stream value
    pp.closure.n_key_fields = 1;
    pp.closure.key_fields[0] = mzgpu_field{MZGPU_SRC_KEY, 0, 64, 0};
    pp.closure.n_val_fields = 1;
    pp.closure.val_fields[0] = mzgpu_field{MZGPU_SRC_VAL2, 0, 64, 0};
  }
  const bool bounded = exact && fan > 0 && n_ub <= MZ_BOUND_MAX_ROWS / fan &&
                       mz_probe_tiles(n_ub, tv.n_batches) <= MZ_LB_TILES;
  if (bounded) {
    const u64 bound = n_ub * fan;
    if (!consolidate_output) {
      MZ_TRY(buf_reserve(out, out->ub + bound, true));
      Append a;
      MZ_TRY(buf_begin_append(out, &a));
      MZ_TRY(mz_probe_async(ctx, d_stream, n, n_ub, tv, pp, out->mem.as<u64>(), a.base, out->cap, a.out_len));
      buf_end_append(out, a, bound);
      return MZGPU_OK;
    }
    // probe into a scratch array, consolidate that, append
    DevMem res, cons;
    Lazy4 rlen, clen;
    u64 ccap = 0;
    MZ_TRY(res.alloc(ctx, bound * 32));
    MZ_TRY(rlen.make_pending(ctx));
    MZ_TRY(mz_probe_async(ctx, d_stream, n, n_ub, tv, pp, res.as<u64>(), dlen_imm(0), bound, rlen.dptr()));
    rlen.mark_written();
    MZ_TRY(consolidate_dev(ctx, 32, res.p, dlen_of(rlen, 0), bound, &cons, &ccap, &clen));
    return buf_append_dev(out, cons.p, dlen_of(clen, 0), clen.known ? clen.v[0] : bound);
  }
  // exact two-pass form
  u64 nn = n.imm;
  if (n.p != nullptr) {
    MZ_TRY(mz_resolve_counters(ctx));
    nn = ctx->h_cnt[n.p - ctx->d_cnt];
  }
  if (nn == 0) return MZGPU_OK;
  DevMem res;
  u64 n_res = 0;
  MZ_TRY(mz_probe(ctx, d_stream, nn, tv, pp, &res, &n_res));
  if (consolidate_output && n_res) {
    DevMem cons;
    Lazy4 clen;
    u64 ccap = 0;
    MZ_TRY(consolidate_dev(ctx, 32, res.p, dlen_imm(n_res), n_res, &cons, &ccap, &clen));
    MZ_TRY(buf_append_dev(out, cons.p, dlen_of(clen, 0), clen.known ? clen.v[0] : n_res));
  } else if (n_res) {
    MZ_TRY(buf_append_dev(out, res.p, dlen_imm(n_res), n_res));
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_half_join(mzgpu_ctx* ctx, const mzgpu_r32* stream, uint64_t n, int32_t mem,
                                   mzgpu_spine* trace, int32_t cmp_mode, const mzgpu_closure* closure,
                                   int32_t consolidate_output, mzgpu_buf* out) {
  MZ_CHECK_CTX(ctx);
  if (trace == nullptr || out == nullptr || (stream == nullptr && n) || trace->rb != 32 || out->rb != 32 ||
      (cmp_mode != MZGPU_HALFJOIN_LE && cmp_mode != MZGPU_HALFJOIN_LT))
    return MZGPU_E_INVALID;
  MZ_TRY(validate_closure(ctx, closure));
  if (n == 0) return MZGPU_OK;
  ctx->stats.rows_in += n;
  DevMem in;
  const u64* d_stream = (const u64*)stream;
  if (mem == MZGPU_MEM_HOST) {
    MZ_TRY(in.alloc(ctx, n * 32));
    MZ_TRY(copy_in(ctx, in.p, stream, n * 32, mem));
    d_stream = in.as<u64>();
  }
  return half_join_dev(ctx, d_stream, dlen_imm(n), n, trace, cmp_mode, closure, consolidate_output, out);
}
// k half joins in one launch (mz_probe_async_many).  Requests whose output buffers coincide must
// be adjacent: they form a chain whose results are appended in request order -- the last stage of
// the delta paths, whose outputs are concatenated (delta_join.rs:302-308).  Anything the single
// launch cannot take (unbounded fan-out, an empty stream or trace, a buffer named twice apart)
// runs request by request; the results are the same either way.
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
};
static int32_t map_rows_into(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const mzgpu_closure* closure,
                             u64 skip_time, mzgpu_buf* out);
static const u64* req_rows(const HalfJoinReq& r) { return r.src ? r.src->rows.as<u64>() : r.stream->mem.as<u64>(); }
static DLen req_dlen(const HalfJoinReq& r) { return r.src ? batch_dlen(r.src) : buf_dlen(r.stream); }
static u64 req_ub(const HalfJoinReq& r) { return r.src ? r.src->len_ub : r.stream->ub; }
static int32_t half_join_many_dev(mzgpu_ctx* ctx, int k, const HalfJoinReq* reqs) {
  auto one_by_one = [&]() -> int32_t {
    for (int j = 0; j < k; ++j) {
      const HalfJoinReq& r = reqs[j];
      if (r.src != nullptr) {
        // the separate operators: update stream into a scratch buffer, then the half join
        mzgpu_buf tmp;
        tmp.ctx = ctx;
        tmp.rb = 32;
        tmp.len.set(ctx, 0);
        MZ_TRY(map_rows_into(ctx, req_rows(r), req_dlen(r), req_ub(r), r.pre, r.skip_time, &tmp));
        MZ_TRY(half_join_dev(ctx, tmp.mem.as<u64>(), buf_dlen(&tmp), tmp.ub, r.trace, r.cmp_mode, r.closure, 0, r.out));
      } else {
        MZ_TRY(half_join_dev(ctx, req_rows(r), req_dlen(r), req_ub(r), r.trace, r.cmp_mode, r.closure, 0, r.out));
      }
    }
    return MZGPU_OK;
  };
  for (int j = 0; j < k; ++j)
    if (reqs[j].src != nullptr) MZ_TRY(batch_ready(reqs[j].src));
  bool any_src = false;
  for (int j = 0; j < k; ++j) any_src = any_src || reqs[j].src != nullptr;
  if ((k < 2 && !any_src) || k > MZ_PROBE_MANY_MAX) return one_by_one();
  static thread_local TraceView tvs[MZ_PROBE_MANY_MAX];  // large: kept off the stack
  ProbeParams pps[MZ_PROBE_MANY_MAX];
  u64 bound[MZ_PROBE_MANY_MAX];
  u64 tiles = 0;
  for (int j = 0; j < k; ++j) {
    const HalfJoinReq& r = reqs[j];
    for (int i = 0; i + 1 < j; ++i)
      if (reqs[i].out == r.out && reqs[j - 1].out != r.out) return one_by_one();
    for (int i = 0; i < k; ++i)
      if (reqs[i].stream != nullptr && reqs[i].stream == r.out) return one_by_one();
    if (req_ub(r) == 0) return one_by_one();
    std::vector<mzgpu_batch*> all;
    spine_readable(r.trace, all);
    u64 fan = 0;
    bool exact = true;
    MZ_TRY(trace_fanout(all, &fan, &exact));
    MZ_TRY(trace_view(ctx, all, &tvs[j]));
    if (tvs[j].n_batches == 0 || !exact || fan == 0 || req_ub(r) > MZ_BOUND_MAX_ROWS / fan) return one_by_one();
    bound[j] = req_ub(r) * fan;
    tiles += mz_probe_tiles(req_ub(r), tvs[j].n_batches);
    memset(&pps[j], 0, sizeof(ProbeParams));
    pps[j].mode = r.cmp_mode == MZGPU_HALFJOIN_LE ? MZ_PROBE_HALF_LE : MZ_PROBE_HALF_LT;
    pps[j].has_closure = 1;
    if (r.closure) {
      pps[j].closure = *r.closure;
    } else {
      pps[j].closure.n_key_fields = 1;
      pps[j].closure.key_fields[0] = mzgpu_field{MZGPU_SRC_KEY, 0, 64, 0};
      pps[j].closure.n_val_fields = 1;
      pps[j].closure.val_fields[0] = mzgpu_field{MZGPU_SRC_VAL2, 0, 64, 0};
    }
  }
  if (tiles > MZ_LB_TILES) return one_by_one();
  // chains: reserve each output for the sum of its requests' bounds, open one append per chain
  ProbeJobHost jobs[MZ_PROBE_MANY_MAX];
  Append app[MZ_PROBE_MANY_MAX];
  u64 chain_bound[MZ_PROBE_MANY_MAX];
  int chain_first[MZ_PROBE_MANY_MAX];
  int nc = 0;
  for (int j = 0; j < k; ++j) {
    if (j == 0 || reqs[j].out != reqs[j - 1].out) {
      chain_first[nc] = j;
      chain_bound[nc] = 0;
      ++nc;
    }
    chain_bound[nc - 1] += bound[j];
  }
  for (int c = 0; c < nc; ++c) {
    mzgpu_buf* out = reqs[chain_first[c]].out;
    MZ_TRY(buf_reserve(out, out->ub + chain_bound[c], true));
    MZ_TRY(buf_begin_append(out, &app[c]));
  }
  int c = -1;
  for (int j = 0; j < k; ++j) {
    if (j == 0 || reqs[j].out != reqs[j - 1].out) ++c;
    mzgpu_buf* out = reqs[j].out;
    jobs[j].d_stream = req_rows(reqs[j]);
    jobs[j].n = req_dlen(reqs[j]);
    jobs[j].n_ub = req_ub(reqs[j]);
    jobs[j].has_pre = reqs[j].src != nullptr;
    jobs[j].pre = reqs[j].pre;
    jobs[j].skip_time = reqs[j].skip_time;
    jobs[j].trace = &tvs[j];
    jobs[j].pp = &pps[j];
    jobs[j].chain = c;
    jobs[j].d_out = out->mem.as<u64>();
    jobs[j].out_base = app[c].base;
    jobs[j].out_cap = out->cap;
    jobs[j].d_out_len = app[c].out_len;
  }
  MZ_TRY(mz_probe_async_many(ctx, k, jobs));
  for (int cc = 0; cc < nc; ++cc) buf_end_append(reqs[chain_first[cc]].out, app[cc], chain_bound[cc]);
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_half_join_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_buf* const* streams,
                                        mzgpu_spine* const* traces, const int32_t* cmp_modes,
                                        const mzgpu_closure* const* closures, mzgpu_buf* const* outs) {
  MZ_CHECK_CTX(ctx);
  if (k == 0) return MZGPU_OK;
  if (streams == nullptr || traces == nullptr || cmp_modes == nullptr || outs == nullptr || k > 64)
    return MZGPU_E_INVALID;
  std::vector<HalfJoinReq> reqs(k);
  for (uint32_t j = 0; j < k; ++j) {
    if (streams[j] == nullptr || traces[j] == nullptr || outs[j] == nullptr || streams[j] == outs[j] ||
        streams[j]->rb != 32 || traces[j]->rb != 32 || outs[j]->rb != 32 ||
        (cmp_modes[j] != MZGPU_HALFJOIN_LE && cmp_modes[j] != MZGPU_HALFJOIN_LT))
      return MZGPU_E_INVALID;
    reqs[j].stream = streams[j];
    reqs[j].trace = traces[j];
    reqs[j].cmp_mode = cmp_modes[j];
    reqs[j].closure = closures ? closures[j] : nullptr;
    MZ_TRY(validate_closure(ctx, reqs[j].closure));
    reqs[j].out = outs[j];
    ctx->stats.rows_in += streams[j]->ub;
  }
  // groups of at most MZ_PROBE_MANY_MAX, never splitting a chain's adjacency
  for (uint32_t at = 0; at < k; at += MZ_PROBE_MANY_MAX) {
    const int g = (int)std::min<uint32_t>(MZ_PROBE_MANY_MAX, k - at);
    MZ_TRY(half_join_many_dev(ctx, g, reqs.data() + at));
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_delta_first_stage_many(mzgpu_ctx* ctx, uint32_t k, mzgpu_batch* const* batches,
                                                const mzgpu_closure* const* initial_closures,
                                                const uint64_t* skip_times, mzgpu_spine* const* traces,
                                                const int32_t* cmp_modes, const mzgpu_closure* const* closures,
                                                mzgpu_buf* const* outs) {
  MZ_CHECK_CTX(ctx);
  if (k == 0) return MZGPU_OK;
  if (batches == nullptr || skip_times == nullptr || traces == nullptr || cmp_modes == nullptr || outs == nullptr ||
      k > 64)
    return MZGPU_E_INVALID;
  std::vector<HalfJoinReq> reqs(k);
  for (uint32_t j = 0; j < k; ++j) {
    if (batches[j] == nullptr || traces[j] == nullptr || outs[j] == nullptr || batches[j]->rb != 32 ||
        traces[j]->rb != 32 || outs[j]->rb != 32 ||
        (cmp_modes[j] != MZGPU_HALFJOIN_LE && cmp_modes[j] != MZGPU_HALFJOIN_LT))
      return MZGPU_E_INVALID;
    reqs[j].stream = nullptr;
    reqs[j].src = batches[j];
    reqs[j].pre = initial_closures ? initial_closures[j] : nullptr;
    reqs[j].skip_time = skip_times[j];
    reqs[j].trace = traces[j];
    reqs[j].cmp_mode = cmp_modes[j];
    reqs[j].closure = closures ? closures[j] : nullptr;
    MZ_TRY(validate_closure(ctx, reqs[j].pre));
    MZ_TRY(validate_closure(ctx, reqs[j].closure));
    reqs[j].out = outs[j];
    ctx->stats.rows_in += batches[j]->len_ub;
  }
  for (uint32_t at = 0; at < k; at += MZ_PROBE_MANY_MAX) {
    const int g = (int)std::min<uint32_t>(MZ_PROBE_MANY_MAX, k - at);
    MZ_TRY(half_join_many_dev(ctx, g, reqs.data() + at));
  }
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_half_join_buf(mzgpu_ctx* ctx, mzgpu_buf* stream, mzgpu_spine* trace, int32_t cmp_mode,
                                       const mzgpu_closure* closure, int32_t consolidate_output, mzgpu_buf* out) {
  MZ_CHECK_CTX(ctx);
  if (stream == nullptr || trace == nullptr || out == nullptr || stream == out || stream->rb != 32 ||
      trace->rb != 32 || out->rb != 32 || (cmp_mode != MZGPU_HALFJOIN_LE && cmp_mode != MZGPU_HALFJOIN_LT))
    return MZGPU_E_INVALID;
  MZ_TRY(validate_closure(ctx, closure));
  ctx->stats.rows_in += stream->ub;
  return half_join_dev(ctx, stream->mem.as<u64>(), buf_dlen(stream), stream->ub, trace, cmp_mode, closure,
                       consolidate_output, out);
}

// rows -> closure(rows) appended to `out`; at most one output row per input row
static int32_t map_rows_into(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const mzgpu_closure* closure,
                             u64 skip_time, mzgpu_buf* out) {
  if (n_ub == 0) return MZGPU_OK;
  if ((n_ub + 255) / 256 > MZ_LB_TILES) {
    u64 nn = n.imm;
    if (n.p != nullptr) {
      MZ_TRY(mz_resolve_counters(ctx));
      nn = ctx->h_cnt[n.p - ctx->d_cnt];
    }
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
struct mzgpu_reduce {
  mzgpu_ctx* ctx;
  int agg_kind;
  TopKParams topk = {-1, 0, 0};
  // mzgpu_reduce_lanes_new: lane class (1, 2, 4, 8) and descriptors; 0 for every other operator
  int lane_class = 0;
  LaneSet lanes = {};
  mzgpu_batcher* batcher = nullptr;
  mzgpu_spine* input = nullptr;
  // distinct lanes (MZGPU_ACCUM_DISTINCT), in lane order: the lane index, and the batcher and R32 pair
  // arrangement of its (key, value) pairs
  int n_distinct = 0;
  u32 distinct_lane[MZGPU_MAX_ACCUM_LANES] = {};
  mzgpu_batcher* pair_batcher[MZGPU_MAX_ACCUM_LANES] = {};
  mzgpu_spine* pairs[MZGPU_MAX_ACCUM_LANES] = {};
  int32_t failed = MZGPU_OK;  // set when an activation failed after its seal (reduce_dev)
  std::string failed_msg;
  ~mzgpu_reduce() {
    delete batcher;
    delete input;
    for (int j = 0; j < n_distinct; ++j) {
      delete pair_batcher[j];
      delete pairs[j];
    }
  }
};

extern "C" int32_t mzgpu_reduce_new(mzgpu_ctx* ctx, int32_t agg_kind, mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || agg_kind < MZGPU_AGG_COUNT_SUM_I64 || agg_kind > MZGPU_AGG_MAX) return MZGPU_E_INVALID;
  std::unique_ptr<mzgpu_reduce> r(new mzgpu_reduce());
  r->ctx = ctx;
  r->agg_kind = agg_kind;
  // accumulable kinds arrange exploded diffs (RACC); MIN/MAX arranges the (key, value) rows themselves
  const uint32_t rb = (agg_kind == MZGPU_AGG_MIN || agg_kind == MZGPU_AGG_MAX) ? 32 : 80;
  MZ_TRY(mzgpu_batcher_new(ctx, rb, &r->batcher));
  MZ_TRY(mzgpu_spine_new(ctx, rb, 1, &r->input));
  *out = r.release();
  return MZGPU_OK;
}
extern "C" int32_t mzgpu_topk_new(mzgpu_ctx* ctx, int64_t limit, uint64_t offset, int32_t descending,
                                  mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr) return MZGPU_E_INVALID;
  std::unique_ptr<mzgpu_reduce> r(new mzgpu_reduce());
  r->ctx = ctx;
  r->agg_kind = MZGPU_AGG_TOPK;
  r->topk.limit = limit < 0 ? -1 : limit;
  r->topk.offset = offset;
  r->topk.descending = descending != 0;
  MZ_TRY(mzgpu_batcher_new(ctx, 32, &r->batcher));
  MZ_TRY(mzgpu_spine_new(ctx, 32, 1, &r->input));
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
  const int c = r->lane_class;
  MZ_TRY(s.rows.alloc(ctx, cap * mz_lane_arr_bytes(c)));
  MZ_TRY(mz_distinct_presence(ctx, c, d, jobs, s.rows.as<u64>(), cap, &s.len, &s.word));
  s.ub = cap;
  return batcher_push_seg(r->batcher, std::move(s));
}

static int32_t reduce_main(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out,
                           bool minmax, u64 per_row);
static int32_t reduce_dev(mzgpu_reduce* r, const u64* d_rows, DLen n, u64 n_ub, u64 upper, mzgpu_buf* out) {
  mzgpu_ctx* ctx = r->ctx;
  if (r->failed != MZGPU_OK) {  // an earlier activation lost its corrections: the operator is dead, not the worker
    ctx->last_error = r->failed_msg;
    return r->failed;
  }
  // batches sealed by earlier activations are merge-eligible now; their lengths
  // have reached the host with whatever the caller read since (no extra wait)
  MZ_TRY(mzgpu_spine_set_physical_compaction(r->input, r->input->upper));
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
      int32_t ins = MZGPU_OK;
      if (pair_new[j]->desc.lower != pair_new[j]->desc.upper) ins = mzgpu_spine_insert(r->pairs[j], pair_new[j]);
      mzgpu_batch_release(pair_new[j]);
      pair_new[j] = nullptr;
      if (st == MZGPU_OK) st = ins;
    }
    if (st != MZGPU_OK && pairs_sealed && !ctx->sticky && r->failed == MZGPU_OK) {
      r->failed = st;
      r->failed_msg = ctx->last_error;
    }
    return st;
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
  // a lanes operator whose lanes are all distinct has no plain explode
  const bool plain = r->lane_class == 0 || r->lanes.distinct_mask != (1u << r->lanes.n) - 1;
  if (n_ub && plain) {
    Seg s;
    if (minmax) {
      MZ_TRY(s.rows.alloc(ctx, n_ub * 32));
      MZ_CUDA(ctx, cudaMemcpyAsync(s.rows.p, d_rows, n_ub * 32, cudaMemcpyDeviceToDevice, ctx->stream));
    } else {
      const int c = r->lane_class;
      MZ_TRY(s.rows.alloc(ctx, n_ub * (c ? mz_lane_arr_bytes(c) : 80)));
      if (c)
        MZ_TRY(mz_explode_lanes(ctx, c, d_rows, n, n_ub, r->lanes, s.rows.as<u64>()));
      else
        MZ_TRY(mz_explode(ctx, d_rows, n, n_ub, r->agg_kind, s.rows.as<u64>()));
    }
    if (n.p == nullptr) {
      s.len.set(ctx, n.imm);
      s.ub = n.imm;
    } else {
      // same count as the input rows: share nothing, copy the word on the device
      MZ_TRY(s.len.make_pending(ctx));
      MZ_CUDA(ctx, cudaMemcpyAsync(s.len.dptr(), n.p, 8, cudaMemcpyDeviceToDevice, ctx->stream));
      s.len.mark_written();
      s.ub = n_ub;
    }
    MZ_TRY(batcher_push_seg(r->batcher, std::move(s)));
  }
  // arrange: seal the accumulable arrangement's batch at the new frontier
  mzgpu_batch* batch = nullptr;
  MZ_TRY(batcher_seal(r->batcher, upper, &batch, nullptr));
  // reduce_abelian over the keys of the new batch
  std::vector<mzgpu_batch*> prior;
  r->input->all_batches(prior);
  TraceView tv;
  int32_t st = trace_view(ctx, prior, &tv);
  const u64 b_ub = batch->len_ub;
  const int lc = r->lane_class ? r->lane_class : 1;
  const u64 out_rb = (u64)mz_lane_out_bytes(lc);
  const LaneSet* ls = r->lane_class ? &r->lanes : nullptr;
  if (st == MZGPU_OK && b_ub > 0) {
    if ((b_ub + 255) / 256 <= MZ_LB_TILES && per_row * b_ub <= MZ_BOUND_MAX_ROWS) {
      DevMem corr, cons;
      Lazy4 clen, flen;
      u64 ccap = 0;
      st = corr.alloc(ctx, per_row * b_ub * out_rb);
      if (st == MZGPU_OK) st = clen.make_pending(ctx);
      if (st == MZGPU_OK) {
        if (minmax)
          st = mz_reduce_minmax_async(ctx, batch->rows.as<u64>(), batch_dlen(batch), b_ub, tv, r->agg_kind,
                                      r->topk, corr.as<u64>(), per_row * b_ub, clen.dptr());
        else
          st = mz_reduce_corrections_async(ctx, lc, batch->rows.as<u64>(), batch_dlen(batch), b_ub, tv,
                                           r->agg_kind, ls, corr.as<u64>(), per_row * b_ub, clen.dptr());
        clen.mark_written();
      }
      if (st == MZGPU_OK && !minmax) {
        // the accumulable kinds' corrections leave the kernel consolidated (reduce.cu:
        // sort_key_corrections): keys ascending, each key's few rows sorted by its thread
        st = buf_append_dev(out, corr.p, dlen_of(clen, 0), per_row * b_ub);
      } else {
        if (st == MZGPU_OK)
          st = consolidate_dev(ctx, 64, corr.p, dlen_of(clen, 0), per_row * b_ub, &cons, &ccap, &flen);
        if (st == MZGPU_OK)
          st = buf_append_dev(out, cons.p, dlen_of(flen, 0), flen.known ? flen.v[0] : per_row * b_ub);
      }
    } else {
      DevMem corr, cons;
      u64 n_corr = 0, ccap = 0;
      Lazy4 flen;
      st = batch_resolve(batch);
      if (st == MZGPU_OK && minmax) {
        MZ_SET_ERR(ctx, "MIN/MAX/TopK reduce: batch of %llu rows exceeds the single-pass bound",
                   (unsigned long long)b_ub);
        st = MZGPU_E_UNSUPPORTED;
      }
      if (st == MZGPU_OK)
        st = mz_reduce_corrections(ctx, lc, batch->rows.as<u64>(), batch->st.v[0], tv, r->agg_kind, ls, &corr,
                                   &n_corr);
      if (st == MZGPU_OK && n_corr && lc > 1) {
        // consolidated by construction, as in the single-pass form (and no RowT for these widths)
        st = buf_append_dev(out, corr.p, dlen_imm(n_corr), n_corr);
      } else {
        if (st == MZGPU_OK && n_corr)
          st = consolidate_dev(ctx, 64, corr.p, dlen_imm(n_corr), n_corr, &cons, &ccap, &flen);
        if (st == MZGPU_OK && n_corr)
          st = buf_append_dev(out, cons.p, dlen_of(flen, 0), flen.known ? flen.v[0] : n_corr);
      }
    }
  }
  // The seal above consumed the batcher's rows and advanced its frontier, so the batch joins the
  // input trace whatever happened since (the arrangement stays consistent with the frontier); a
  // failure after the seal means this activation's corrections are missing from `out`, which no
  // later activation can repair: the operator reports that status from now on.
  int32_t ins = MZGPU_OK;
  if (batch->desc.lower != batch->desc.upper) ins = mzgpu_spine_insert(r->input, batch);
  mzgpu_batch_release(batch);
  if (st == MZGPU_OK) st = ins;
  if (st != MZGPU_OK && !ctx->sticky) {
    r->failed = st;
    r->failed_msg = ctx->last_error;
  }
  return st;
}

extern "C" int32_t mzgpu_reduce_accumulable(mzgpu_reduce* r, const mzgpu_r32* rows, uint64_t n,
                                            int32_t mem, uint64_t upper, mzgpu_buf* out) {
  if (r == nullptr || out == nullptr || (rows == nullptr && n) || out->rb != 64 || r->lane_class) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = r->ctx;
  MZ_CHECK_CTX(ctx);
  ctx->stats.rows_in += n;
  DevMem in;
  const u64* d_rows = (const u64*)rows;
  if (mem == MZGPU_MEM_HOST && n) {
    MZ_TRY(in.alloc(ctx, n * 32));
    MZ_TRY(copy_in(ctx, in.p, rows, n * 32, mem));
    d_rows = in.as<u64>();
  }
  return reduce_dev(r, d_rows, dlen_imm(n), n, upper, out);
}
extern "C" int32_t mzgpu_reduce_accumulable_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper,
                                                mzgpu_buf* out) {
  if (r == nullptr || rows == nullptr || out == nullptr || rows->rb != 32 || out->rb != 64 || r->lane_class)
    return MZGPU_E_INVALID;
  MZ_CHECK_CTX(r->ctx);
  r->ctx->stats.rows_in += rows->ub;
  return reduce_dev(r, rows->mem.as<u64>(), buf_dlen(rows), rows->ub, upper, out);
}

// ------------------------------------------------------- reduce over several value columns
extern "C" int32_t mzgpu_reduce_lanes_row_bytes(uint32_t n_lanes, uint32_t* arr_row_bytes, uint32_t* out_row_bytes) {
  if (n_lanes == 0 || n_lanes > MZGPU_MAX_ACCUM_LANES) return MZGPU_E_INVALID;
  const int c = mz_lane_class(n_lanes);
  if (arr_row_bytes != nullptr) *arr_row_bytes = (uint32_t)mz_lane_arr_bytes(c);
  if (out_row_bytes != nullptr) *out_row_bytes = (uint32_t)mz_lane_out_bytes(c);
  return MZGPU_OK;
}

extern "C" int32_t mzgpu_reduce_lanes_new(mzgpu_ctx* ctx, uint32_t in_row_bytes, const mzgpu_accum_lane* lanes,
                                          uint32_t n_lanes, mzgpu_reduce** out) {
  MZ_CHECK_CTX(ctx);
  if (out == nullptr || (lanes == nullptr && n_lanes) || (in_row_bytes != 32 && in_row_bytes != 40)) {
    MZ_SET_ERR(ctx, "reduce_lanes: bad arguments (input rows of %u bytes)", in_row_bytes);
    return MZGPU_E_INVALID;
  }
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
    const char* bad = nullptr;
    if (base != MZGPU_AGG_COUNT_SUM_I64 && !f64)
      bad = "kind is not COUNT_SUM_I64 / COUNT_SUM_F64, optionally | MZGPU_ACCUM_DISTINCT";
    else if (f.src != MZGPU_SRC_VAL1 && !(f.src == MZGPU_SRC_VAL2 && in_row_bytes == 40))
      bad = "source word is not a value word of the input row";
    else if (f.bits == 0 || f.bits > 64 || f.shift > 63 || (u32)f.shift + f.bits > 64)
      bad = "field is empty or out of range";
    else if (f64 && (f.shift != 0 || f.bits != 64))
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
  std::unique_ptr<mzgpu_reduce> r(new mzgpu_reduce());
  r->ctx = ctx;
  r->lane_class = mz_lane_class(n_lanes);
  r->lanes = ls;
  // class 1 runs the one-column kernels, which take the lane's kind (without the DISTINCT bit) as the
  // aggregate kind
  r->agg_kind = (ls.f64_mask & 1u) ? MZGPU_AGG_COUNT_SUM_F64 : MZGPU_AGG_COUNT_SUM_I64;
  const uint32_t rb = (uint32_t)mz_lane_arr_bytes(r->lane_class);
  MZ_TRY(mzgpu_batcher_new(ctx, rb, &r->batcher));
  MZ_TRY(mzgpu_spine_new(ctx, rb, 1, &r->input));
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

extern "C" mzgpu_spine* mzgpu_reduce_lanes_distinct_trace(mzgpu_reduce* r, uint32_t lane) {
  if (r == nullptr) return nullptr;
  for (int j = 0; j < r->n_distinct; ++j)
    if (r->distinct_lane[j] == lane) return r->pairs[j];
  return nullptr;
}

static bool lanes_io_ok(mzgpu_reduce* r, uint32_t in_rb, mzgpu_buf* out) {
  return r->lane_class != 0 && in_rb == r->lanes.in_words * 8 && out->rb == (uint32_t)mz_lane_out_bytes(r->lane_class);
}
extern "C" int32_t mzgpu_reduce_lanes(mzgpu_reduce* r, const void* rows, uint64_t n, int32_t mem, uint64_t upper,
                                      mzgpu_buf* out) {
  if (r == nullptr || out == nullptr || (rows == nullptr && n)) return MZGPU_E_INVALID;
  mzgpu_ctx* ctx = r->ctx;
  MZ_CHECK_CTX(ctx);
  const uint32_t in_rb = r->lanes.in_words * 8;
  if (!lanes_io_ok(r, in_rb, out)) {
    MZ_SET_ERR(ctx, "reduce_lanes: output buffer of %u-byte rows", out->rb);
    return MZGPU_E_INVALID;
  }
  ctx->stats.rows_in += n;
  DevMem in;
  const u64* d_rows = (const u64*)rows;
  if (mem == MZGPU_MEM_HOST && n) {
    MZ_TRY(in.alloc(ctx, n * in_rb));
    MZ_TRY(copy_in(ctx, in.p, rows, n * in_rb, mem));
    d_rows = in.as<u64>();
  }
  return reduce_dev(r, d_rows, dlen_imm(n), n, upper, out);
}
extern "C" int32_t mzgpu_reduce_lanes_buf(mzgpu_reduce* r, mzgpu_buf* rows, uint64_t upper, mzgpu_buf* out) {
  if (r == nullptr || rows == nullptr || out == nullptr) return MZGPU_E_INVALID;
  MZ_CHECK_CTX(r->ctx);
  if (!lanes_io_ok(r, rows->rb, out)) {
    MZ_SET_ERR(r->ctx, "reduce_lanes: input rows of %u bytes / output rows of %u bytes", rows->rb, out->rb);
    return MZGPU_E_INVALID;
  }
  r->ctx->stats.rows_in += rows->ub;
  return reduce_dev(r, rows->mem.as<u64>(), buf_dlen(rows), rows->ub, upper, out);
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
