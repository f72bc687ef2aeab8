// common.cuh — context, device memory, row traits and block-level primitives
// shared by every kernel file of libmzgpu (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <chrono>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/mzgpu.h"

typedef uint64_t u64;
typedef int64_t i64;
typedef uint32_t u32;

// ------------------------------------------------------------------ errors
struct mzgpu_ctx {
  int device = 0;
  int worker = 0;
  int peers = 1;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev = nullptr;
  cudaEvent_t ev_block = nullptr;  // MZGPU_BLOCKING_SYNC=1: host waits block on this event (no spinning)
  int num_sms = 132;
  bool sticky = false;  // a CUDA/NCCL failure (or a deferred device-side report) happened: every later call fails
  int32_t sticky_code = MZGPU_E_CUDA;  // ... with this status
  std::string last_error;
  mzgpu_stats stats;
  // pinned staging for small device->host reads (counts, min/max)
  u64* h_scratch = nullptr;  // 64 words
  u64* d_scratch = nullptr;  // 64 words
  u64* h_big = nullptr;      // pinned, 512 words (exchange counts)
  u64 last_minmax[14] = {0};  // min/max of every key word seen by the last bulk sort (mz_sort_perm)
  bool last_minmax_valid = false;
  // pinned bounce buffers for host<->device row copies
  void* h_bounce = nullptr;
  size_t h_bounce_bytes = 0;
  // ---- device-resident counters (lazy read-back; see Lazy4 below)
  u64* d_cnt = nullptr;        // MZ_CNT_BLOCKS x 4 words
  u64* h_cnt = nullptr;        // pinned mirror, refreshed by mz_resolve_counters()
  std::vector<int> cnt_free;   // free block indices
  std::vector<int> cnt_parked; // freed while side-stream work was outstanding: reusable after the join
  int cnt_high = 0;            // blocks [0, cnt_high) have been handed out at least once
  u64 op_seq = 1;              // bumped whenever a kernel that writes counters is enqueued
  u64 resolved_seq = 0;        // op_seq covered by the last read-back
  u64 n_resolves = 0;          // host syncs spent on read-backs
  u64 ns_alloc = 0, ns_sync = 0, n_alloc = 0, bytes_alloc = 0;  // host-side time in the allocator / waiting (MZGPU_DEBUG)
  // ---- single-pass expansion kernels: look-back state, tile tickets
  u64* d_lb = nullptr;         // MZ_LB_TILES tagged state words (never written by anything else)
  u32 lb_epoch = 0;            // tag of the next launch (20 bits)
  u32* d_tickets = nullptr;    // MZ_TICKETS zeroed tile counters, handed out round-robin
  u32 ticket_next = 0;
  // the same for single-pass kernels launched on the side stream (they run concurrently with the main
  // stream's: shared state words or a shared ticket reset would corrupt each other)
  u64* d_lb_side = nullptr;
  u32* d_tickets_side = nullptr;
  u32 ticket_next_side = 0;
  // merges in flight on the side stream whose inputs readers still use (host.cu: mz_join_side)
  std::vector<struct mzgpu_batch*> side_outputs;
  u64* d_status = nullptr;     // [0] != 0: a bounded output overflowed (rows required), [1] != 0: a MIN/MAX key outgrew its table
  u64* d_dbg = nullptr;  // per-launch phase stamps of the fused kernel while profiling (32 words each)
  u32 dbg_next = 0;
  // control blocks of the fused kernel, a pair per stream (each launch clears the other of its pair)
  void* d_fused_ctl[4] = {nullptr, nullptr, nullptr, nullptr};
  int fused_flip[2] = {0, 0};
  void* d_fused_ctl_many[16] = {};  // per job slot: 0-3 multi-job launches, 4-7 deferred jobs
  int fused_flip_many[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  void* fused_deferred = nullptr;       // fused.cu: jobs prepared but not launched yet
  std::vector<struct mzgpu_batch*> deferred_inputs;  // retained until the flush
  u64 defer_seq = 0, flushed_seq = 0;   // deferred jobs enqueued / launched
  int deferred_unlaunched = 0;          // jobs prepared by mz_fused_defer and not launched yet
  // ---- side stream: batch merges (spine maintenance) run here, concurrently with the
  // operators on the main stream; a batch produced here carries side_seq and the main
  // stream waits for the side stream the first time it touches such a batch
  cudaStream_t main_stream = nullptr, side_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_side = nullptr;
  u64 side_seq = 0;    // merges issued on the side stream so far
  u64 joined_seq = 0;  // the main stream has waited for merges <= this
  // per-kernel profiling (mzgpu_profile_enable)
  struct ProfRec {
    const char* name;
    cudaEvent_t e0, e1;
    u64 bytes;
  };
  bool profile = false;
  u64 next_bytes = 0;  // algorithmic bytes of the next launch (MZ_BYTES)
  std::vector<ProfRec> prof;
  std::vector<cudaEvent_t> ev_pool;
  // NCCL (resolved with dlopen at mzgpu_comm_init)
  void* nccl_lib = nullptr;
  void* nccl_comm = nullptr;
  // exchange over peer memory (exchange.cu): landing zones, one per worker
  void* p2p_local = nullptr;        // this worker's zone (cudaMalloc: IPC-exportable)
  void* p2p_peer[16] = {};          // every worker's zone as mapped here ([worker] == p2p_local)
  bool p2p_peer_ipc[16] = {};       // mapped with cudaIpcOpenMemHandle (closed at destroy)
  u64 p2p_rows = 0;                 // rows per region
  u32 p2p_region_rb = 0;            // bytes per row reserved in a region
  u64 p2p_round = 0;                // rounds issued so far
  u64* p2p_cursors = nullptr;       // [MZ_MAX_EXCHANGE][16] scatter cursors (zero between rounds)
  u32* p2p_done = nullptr;          // scatter CTAs finished (zero between rounds)
  bool p2p_ready = false;
  // large blocks (>= MZ_BIG_BLOCK bytes) freed by this ctx, kept for reuse (DevMem): the bulk regimes
  // (hydration, BASELINE configs 1/2/4) cycle through a handful of multi-GB arrays per call
  struct BigBlock {
    void* p;
    size_t bytes;
    cudaStream_t freed_on;  // the ctx stream at the time of the free
    unsigned ok;            // mid-size blocks: streams whose order already covers the free (1 main, 2 side)
  };
  std::vector<BigBlock> big_cache;
  size_t big_cached_bytes = 0;
  u64 big_hits = 0, big_misses = 0;
  // mid-size blocks ([mid_block, MZ_BIG_BLOCK)): kept too, and handed out again only to a stream whose order
  // already covers the free -- the stream it was freed on, the side stream once it has forked from the main
  // stream after the free, the main stream once it has joined the side stream after the free (mz_mid_forked /
  // mz_mid_joined) -- so no event wait is ever added: merges and operators stay decoupled
  std::vector<BigBlock> mid_cache;
  size_t mid_cached_bytes = 0;
  u64 mid_hits = 0, mid_misses = 0;
  size_t mid_block = (size_t)8 << 20;  // MZGPU_MID_BLOCK_MB (0: off)
};
// Blocks of at least this size bypass the driver's stream-ordered pool on reuse: cudaMallocAsync of
// multi-GB blocks can cost host time that grows from call to call (tools/diag_bulk.py cfg4 shows it for
// the 100M-row reduce) although every block was freed in stream order before.  The update-batch path
// (blocks of a few hundred MB at most) allocates in microseconds and stays on the pool.  The cache holds
// at most half of the H100's 80 GB; an allocation that fails hands every cached block back first.
#define MZ_BIG_BLOCK ((size_t)512 << 20)
#define MZ_BIG_CACHE_MAX ((size_t)40 << 30)
// Mid-size blocks: with several workers an operator's scratch is sized by what the worker COULD receive
// (a reduce activation at 2 GPUs allocates and frees ~600 MB in blocks of 30-200 MB for ~10 K actual rows),
// and the driver's pool spends host time on every such cudaMallocAsync / cudaFreeAsync on the hot path.
#define MZ_MID_CACHE_MAX ((size_t)8 << 30)
// the side stream has just been made to wait for the main stream: what the main stream's order covers, the
// side stream's order covers now
static inline void mz_mid_forked(mzgpu_ctx* ctx) {
  for (auto& b : ctx->mid_cache)
    if (b.ok & 1u) b.ok |= 2u;
}
// the main stream has just been made to wait for everything issued on the side stream
static inline void mz_mid_joined(mzgpu_ctx* ctx) {
  for (auto& b : ctx->mid_cache)
    if (b.ok & 2u) b.ok |= 1u;
}

#define MZ_SET_ERR(ctx, ...)                              \
  do {                                                    \
    char _buf[512];                                       \
    snprintf(_buf, sizeof(_buf), __VA_ARGS__);            \
    (ctx)->last_error = _buf;                             \
  } while (0)

#define MZ_CUDA(ctx, expr)                                                               \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      MZ_SET_ERR(ctx, "CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__,      \
                 __LINE__, cudaGetErrorString(_e));                                      \
      (ctx)->sticky = true;                                                              \
      return MZGPU_E_CUDA;                                                               \
    }                                                                                    \
  } while (0)

// a host wait on the ctx stream (counted: mzgpu_stats.host_syncs)
#define MZ_SYNC(ctx)                                            \
  do {                                                          \
    auto _t0 = std::chrono::steady_clock::now();                \
    if ((ctx)->ev_block != nullptr) {                           \
      /* MZGPU_BLOCKING_SYNC=1: sleep in the driver instead of spinning on a core */ \
      MZ_CUDA(ctx, cudaEventRecord((ctx)->ev_block, (ctx)->stream)); \
      MZ_CUDA(ctx, cudaEventSynchronize((ctx)->ev_block));      \
    } else {                                                    \
      MZ_CUDA(ctx, cudaStreamSynchronize((ctx)->stream));       \
    }                                                           \
    (ctx)->ns_sync += (u64)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - _t0).count(); \
    (ctx)->stats.host_syncs++;                                  \
  } while (0)

#define MZ_TRY(expr)                 \
  do {                               \
    int32_t _s = (expr);             \
    if (_s != MZGPU_OK) return _s;   \
  } while (0)

#define MZ_CNT_BLOCKS 8192
#define MZ_LB_TILES (1u << 20)
#define MZ_TICKETS 4096
#define MZ_DBG_RECORDS 4096

#define MZ_CHECK_CTX(ctx)                       \
  do {                                          \
    if ((ctx) == nullptr) return MZGPU_E_INVALID; \
    if ((ctx)->sticky) return (ctx)->sticky_code; \
  } while (0)

// Brackets one launch with CUDA events on the launching stream when profiling.
struct ProfScope {
  mzgpu_ctx* ctx;
  mzgpu_ctx::ProfRec rec;
  bool on;
  ProfScope(mzgpu_ctx* c, const char* name) : ctx(c), on(c->profile) {
    if (!on) return;
    rec.name = name;
    rec.bytes = c->next_bytes;
    for (cudaEvent_t* e : {&rec.e0, &rec.e1}) {
      if (!c->ev_pool.empty()) {
        *e = c->ev_pool.back();
        c->ev_pool.pop_back();
      } else {
        cudaEventCreate(e);
      }
    }
    cudaEventRecord(rec.e0, c->stream);
  }
  ~ProfScope() {
    ctx->next_bytes = 0;
    if (!on) return;
    cudaEventRecord(rec.e1, ctx->stream);
    ctx->prof.push_back(rec);
  }
};
// algorithmic bytes the next launch moves (documented per kernel in DESIGN.md)
#define MZ_BYTES(ctx, n) ((ctx)->next_bytes = (u64)(n))

// Kernel launch helper: counts launches (mzgpu_stats.kernel_launches) and
// surfaces launch-configuration errors immediately.
#define MZ_LAUNCH(ctx, kernel, grid, block, smem, ...)                              \
  do {                                                                              \
    {                                                                               \
      ProfScope _prof(ctx, #kernel);                                                \
      kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);              \
    }                                                                               \
    (ctx)->stats.kernel_launches++;                                                 \
    MZ_CUDA(ctx, cudaGetLastError());                                               \
  } while (0)

// ------------------------------------------------------------ device memory
// Stream-ordered allocations from the device's default mempool (kept warm by a
// release threshold of UINT64_MAX set at ctx creation), with byte accounting
// for the arrangement-size metrics.
struct DevMem {
  mzgpu_ctx* ctx = nullptr;
  void* p = nullptr;
  size_t bytes = 0;
  DevMem() {}
  DevMem(const DevMem&) = delete;
  DevMem& operator=(const DevMem&) = delete;
  DevMem(DevMem&& o) noexcept { *this = std::move(o); }
  DevMem& operator=(DevMem&& o) noexcept {
    if (this != &o) {
      release();
      ctx = o.ctx;
      p = o.p;
      bytes = o.bytes;
      o.p = nullptr;
      o.bytes = 0;
    }
    return *this;
  }
  ~DevMem() { release(); }
  // `exact`: long-lived storage sized to its contents (a shrunk batch) -- never a larger parked block
  int32_t alloc(mzgpu_ctx* c, size_t n, bool exact = false) {
    release();
    ctx = c;
    if (n == 0) n = 16;
    if (n >= MZ_BIG_BLOCK && !exact) {
      // best fit among the cached big blocks, wasting at most half of the block
      int best = -1;
      for (int i = 0; i < (int)c->big_cache.size(); ++i) {
        const size_t b = c->big_cache[i].bytes;
        if (b >= n && b / 2 <= n && (best < 0 || b < c->big_cache[best].bytes)) best = i;
      }
      if (best >= 0) {
        const mzgpu_ctx::BigBlock blk = c->big_cache[best];
        c->big_cache.erase(c->big_cache.begin() + best);
        c->big_cached_bytes -= blk.bytes;
        if (blk.freed_on != c->stream) {
          // freed in another stream's order: everything enqueued there so far happens first
          if (cudaEventRecord(c->ev, blk.freed_on) != cudaSuccess || cudaStreamWaitEvent(c->stream, c->ev, 0) != cudaSuccess) {
            MZ_SET_ERR(c, "big-block reuse: cross-stream ordering failed");
            c->sticky = true;
            return MZGPU_E_CUDA;
          }
        }
        p = blk.p;
        bytes = blk.bytes;
        c->big_hits++;
        c->stats.device_bytes_in_use += bytes;
        if (c->stats.device_bytes_in_use > c->stats.device_bytes_peak)
          c->stats.device_bytes_peak = c->stats.device_bytes_in_use;
        return MZGPU_OK;
      }
      c->big_misses++;
    }
    if (c->mid_block != 0 && n >= c->mid_block && n < MZ_BIG_BLOCK && !exact) {
      // best fit among the blocks whose free this stream's order already covers (no event needed)
      const unsigned me = (c->side_stream != nullptr && c->stream == c->side_stream) ? 2u : 1u;
      int best = -1;
      for (int i = 0; i < (int)c->mid_cache.size(); ++i) {
        const size_t b = c->mid_cache[i].bytes;
        if ((c->mid_cache[i].ok & me) != 0 && b >= n && b / 2 <= n && (best < 0 || b < c->mid_cache[best].bytes))
          best = i;
      }
      if (best >= 0) {
        const mzgpu_ctx::BigBlock blk = c->mid_cache[best];
        c->mid_cache.erase(c->mid_cache.begin() + best);
        c->mid_cached_bytes -= blk.bytes;
        p = blk.p;
        bytes = blk.bytes;
        c->mid_hits++;
        c->stats.device_bytes_in_use += bytes;
        if (c->stats.device_bytes_in_use > c->stats.device_bytes_peak)
          c->stats.device_bytes_peak = c->stats.device_bytes_in_use;
        return MZGPU_OK;
      }
      c->mid_misses++;
    }
    auto t0 = std::chrono::steady_clock::now();
    cudaError_t e = cudaMallocAsync(&p, n, c->stream);
    if (e != cudaSuccess && (!c->big_cache.empty() || !c->mid_cache.empty())) {
      // out of memory with blocks parked in the caches: hand them back (each in the order of the stream
      // it was freed on), let those frees happen, and try once more
      (void)cudaGetLastError();
      for (auto& b : c->big_cache) cudaFreeAsync(b.p, b.freed_on);
      for (auto& b : c->mid_cache) cudaFreeAsync(b.p, b.freed_on);
      c->big_cache.clear();
      c->big_cached_bytes = 0;
      c->mid_cache.clear();
      c->mid_cached_bytes = 0;
      cudaDeviceSynchronize();
      e = cudaMallocAsync(&p, n, c->stream);
    }
    c->ns_alloc += (u64)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
    c->n_alloc++;
    c->bytes_alloc += n;
    if (e != cudaSuccess) {
      p = nullptr;
      MZ_SET_ERR(c, "cudaMallocAsync(%zu bytes) failed: %s", n, cudaGetErrorString(e));
      c->sticky = true;
      return MZGPU_E_CUDA;
    }
    bytes = n;
    c->stats.device_bytes_in_use += n;
    if (c->stats.device_bytes_in_use > c->stats.device_bytes_peak)
      c->stats.device_bytes_peak = c->stats.device_bytes_in_use;
    return MZGPU_OK;
  }
  void release() {
    if (p != nullptr) {
      ctx->stats.device_bytes_in_use -= bytes;
      if (bytes >= MZ_BIG_BLOCK && ctx->big_cached_bytes + bytes <= MZ_BIG_CACHE_MAX) {
        ctx->big_cache.push_back(mzgpu_ctx::BigBlock{p, bytes, ctx->stream, 0u});
        ctx->big_cached_bytes += bytes;
      } else if (ctx->mid_block != 0 && bytes >= ctx->mid_block && bytes < MZ_BIG_BLOCK) {
        ctx->mid_cache.push_back(mzgpu_ctx::BigBlock{
            p, bytes, ctx->stream, (ctx->side_stream != nullptr && ctx->stream == ctx->side_stream) ? 2u : 1u});
        ctx->mid_cached_bytes += bytes;
        // over the budget: the oldest parked blocks go back to the driver's pool, in the order of their stream
        while (ctx->mid_cached_bytes > MZ_MID_CACHE_MAX && ctx->mid_cache.size() > 1) {
          const mzgpu_ctx::BigBlock old = ctx->mid_cache.front();
          ctx->mid_cache.erase(ctx->mid_cache.begin());
          ctx->mid_cached_bytes -= old.bytes;
          cudaFreeAsync(old.p, old.freed_on);
        }
      } else {
        auto t0 = std::chrono::steady_clock::now();
        cudaFreeAsync(p, ctx->stream);
        ctx->ns_alloc += (u64)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
      }
      p = nullptr;
      bytes = 0;
    }
  }
  template <class T>
  T* as() const {
    return (T*)p;
  }
};

// ------------------------------------------------ device-resident row counts
// Data-dependent sizes (rows surviving a consolidation, matches of a probe, ...)
// are produced by kernels.  Reading each one back costs a host sync, and a
// 100K-row update batch is a chain of ~20 such operators whose kernels run for
// microseconds: the syncs, not the kernels, would set the pace.  So a count
// lives in a 4-word block of a small device arena; consumer kernels read it
// from there (DLen), the host works with upper bounds, and the arena is read
// back in one copy the first time the host needs any exact value — which
// resolves every count produced before that point.
int32_t mz_resolve_counters(mzgpu_ctx* ctx);  // host.cu: one D2H of the arena + sync
int mz_cnt_alloc(mzgpu_ctx* ctx);             // -1 if the arena is exhausted
void mz_cnt_free(mzgpu_ctx* ctx, int blk);
void mz_cnt_unpark(mzgpu_ctx* ctx);

struct Lazy4 {
  mzgpu_ctx* ctx = nullptr;
  int blk = -1;
  u64 seq = 0;        // ctx->op_seq when the producing kernel was enqueued
  bool known = true;  // host copy `v` is valid
  u64 v[4] = {0, 0, 0, 0};
  Lazy4() {}
  Lazy4(const Lazy4&) = delete;
  Lazy4& operator=(const Lazy4&) = delete;
  Lazy4(Lazy4&& o) noexcept { *this = std::move(o); }
  Lazy4& operator=(Lazy4&& o) noexcept {
    if (this != &o) {
      drop();
      ctx = o.ctx;
      blk = o.blk;
      seq = o.seq;
      known = o.known;
      for (int i = 0; i < 4; ++i) v[i] = o.v[i];
      o.blk = -1;
      o.known = true;
    }
    return *this;
  }
  ~Lazy4() { drop(); }
  void drop() {
    if (blk >= 0) mz_cnt_free(ctx, blk);
    blk = -1;
  }
  void set(mzgpu_ctx* c, u64 a, u64 b = 0, u64 cc = 0, u64 d = 0) {
    drop();
    ctx = c;
    known = true;
    v[0] = a;
    v[1] = b;
    v[2] = cc;
    v[3] = d;
  }
  // reserve a device block that a kernel enqueued next will fill
  int32_t make_pending(mzgpu_ctx* c) {
    drop();
    ctx = c;
    blk = mz_cnt_alloc(c);
    if (blk < 0) {
      MZ_SET_ERR(c, "device counter arena exhausted (%d blocks unresolved)", MZ_CNT_BLOCKS);
      return MZGPU_E_CAPACITY;
    }
    known = false;
    return MZGPU_OK;
  }
  u64* dptr() const { return ctx->d_cnt + 4 * (size_t)blk; }
  // call right after enqueuing the kernel that writes the block
  void mark_written() { seq = ++ctx->op_seq; }
  // true if the value is known afterwards; never waits for the device
  bool try_resolve() {
    if (known) return true;
    if (seq > ctx->resolved_seq) return false;
    for (int i = 0; i < 4; ++i) v[i] = ctx->h_cnt[4 * (size_t)blk + i];
    known = true;
    drop();
    return true;
  }
  int32_t resolve() {
    if (known) return MZGPU_OK;
    if (seq > ctx->resolved_seq) MZ_TRY(mz_resolve_counters(ctx));
    for (int i = 0; i < 4; ++i) v[i] = ctx->h_cnt[4 * (size_t)blk + i];
    known = true;
    drop();
    return MZGPU_OK;
  }
};

// A row count as a kernel argument: device word if `p`, else the immediate.
struct DLen {
  const u64* p;
  u64 imm;
};
static inline DLen dlen_of(const Lazy4& l, int word) {
  DLen d;
  if (l.known) {
    d.p = nullptr;
    d.imm = l.v[word];
  } else {
    d.p = l.dptr() + word;
    d.imm = 0;
  }
  return d;
}
static inline DLen dlen_imm(u64 n) {
  DLen d;
  d.p = nullptr;
  d.imm = n;
  return d;
}

// Per-launch handle for the single-pass ("chained scan") expansion kernels.
struct LookBack {
  u64* state;   // ctx->d_lb
  u32* ticket;  // one zeroed counter
  u32 epoch;    // tag of this launch
};
int32_t mz_lookback_begin(mzgpu_ctx* ctx, u64 max_tiles, LookBack* lb);  // host.cu
// the same over the state words [at, at + max_tiles): concurrent chains of one launch
int32_t mz_lookback_begin_at(mzgpu_ctx* ctx, u64 at, u64 max_tiles, LookBack* lb);

// ---------------------------------------------------------------- row traits
// A row is NW 64-bit words: NK sort-key words first (compared as unsigned, in
// order), then the diff words.  TW = index of the time word (or -1).  SG = the
// diff's semigroup: MZ_SG_SUM (differences that add, and vanish at zero) or
// MZ_SG_MAX (the monotonic reduce: per-word unsigned max, never zero).
enum : int { MZ_SG_SUM = 0, MZ_SG_MAX = 1 };
template <int RB>
struct RowT;
template <>
struct RowT<16> {  // mzgpu_r16 (key | diff)
  static constexpr int NW = 2, NK = 1, ND = 1, TW = -1, DK = 1, SG = MZ_SG_SUM;
};
template <>
struct RowT<32> {  // mzgpu_r32 (key, val, time | diff)
  static constexpr int NW = 4, NK = 3, ND = 1, TW = 2, DK = 2, SG = MZ_SG_SUM;
};
template <>
struct RowT<40> {  // mzgpu_r40 (key, val1, val2, time | diff)
  static constexpr int NW = 5, NK = 4, ND = 1, TW = 3, DK = 3, SG = MZ_SG_SUM;
};
template <>
struct RowT<80> {  // mzgpu_racc (key, time | total, non_nulls, acc_lo, acc_hi, pinf, ninf, nan, pad)
  static constexpr int NW = 10, NK = 2, ND = 8, TW = 1, DK = 1, SG = MZ_SG_SUM;
};
template <>
struct RowT<64> {  // mzgpu_rout (key, count, sum_lo, sum_hi, flags, time | diff, pad)
  static constexpr int NW = 8, NK = 6, ND = 2, TW = 5, DK = 5, SG = MZ_SG_SUM;
};
// Multi-lane accumulable arrangement rows (mzgpu_reduce_lanes_new): key, time | total, then
// C lanes of (non_nulls, acc_lo, acc_hi, pos_infs, neg_infs, nans), padded to 16 bytes.
template <>
struct RowT<128> {  // C = 2
  static constexpr int NW = 16, NK = 2, ND = 14, TW = 1, DK = 1, SG = MZ_SG_SUM;
};
template <>
struct RowT<224> {  // C = 4
  static constexpr int NW = 28, NK = 2, ND = 26, TW = 1, DK = 1, SG = MZ_SG_SUM;
};
template <>
struct RowT<416> {  // C = 8
  static constexpr int NW = 52, NK = 2, ND = 50, TW = 1, DK = 1, SG = MZ_SG_SUM;
};
// Monotonic MIN / MAX arrangement rows (mzgpu_reduce_monotonic_new): key, time | one encoded lane
// word per lane (MonoRows below), the class's unused lanes and the pad words zero.
template <>
struct RowT<48> {  // 1-4 lanes
  static constexpr int NW = 6, NK = 2, ND = 4, TW = 1, DK = 1, SG = MZ_SG_MAX;
};
template <>
struct RowT<112> {  // 5-8 lanes, 4 pad words
  static constexpr int NW = 14, NK = 2, ND = 12, TW = 1, DK = 1, SG = MZ_SG_MAX;
};
// Monotonic TopK window rows (mzgpu_topk_monotonic_new): key, o0, o1, o2, val1, val2, time | diff, pad.
// o0..o2 are the encoded order lanes (TopKOrder below), so unsigned word order within a key is the
// plan's order, ties broken by (val1, val2).  The only row with more than 6 key words.
template <>
struct RowT<72> {
  static constexpr int NW = 9, NK = 7, ND = 2, TW = 6, DK = 6, SG = MZ_SG_SUM;
};
// DK = number of leading "data" words (key words before the time word): two
// rows with equal DK words are the same (key, val).
//
// Every width has exactly one meaning, because the generic kernels (sort, consolidate, merge,
// index) pick the diff arithmetic from the width alone.  The lanes operator's output rows for
// C >= 2 (96, 144 and 240 bytes, LaneRows below) and the monotonic operator's output rows (56 and
// 88 bytes, MonoRows below) were given widths that no arrangement row uses, and deliberately have
// no RowT: mzgpu_buf_consolidate on them returns MZGPU_E_UNSUPPORTED instead of summing the wrong
// words.

// The compile-time values a runtime row width (or lane class) is dispatched over; each set is named
// once here and every entry point instantiates its kernels for exactly the members of its set.
template <int... V>
struct IntSet {
  static constexpr const char* kind = "row width";
  static constexpr bool has(int v) { return ((v == V) || ...); }
};
using RowWidths = IntSet<16, 32, 40, 64, 80, 128, 224, 416, 48, 112, 72>;  // every RowT: sort, consolidate, fused
// sorted batches: merge, extract, index (40: the hierarchical MIN / MAX reduce arranges its R40 input)
using BatchWidths = IntSet<32, 64, 80, 128, 224, 416, 48, 112, 72, 40>;
using ExchangeWidths = IntSet<32, 80>;
struct LaneClasses : IntSet<1, 2, 4, 8> {  // accumulable reduce with 1, 2, 4 or 8 lanes (LaneRows below)
  static constexpr const char* kind = "lane class";
};

template <int... V, class F>
int32_t mz_dispatch_in(IntSet<V...>, mzgpu_ctx* ctx, int value, const char* what, const char* kind, F&& f) {
  int32_t st = MZGPU_OK;
  if (((value == V && (st = f(std::integral_constant<int, V>()), true)) || ...)) return st;
  MZ_SET_ERR(ctx, "%s: unsupported %s %d", what, kind, value);
  return MZGPU_E_UNSUPPORTED;
}
// f(std::integral_constant<int, value>()) when `value` is a member of Set, and its status;
// MZGPU_E_UNSUPPORTED (with "<what>: unsupported <Set::kind> <value>" as the last error) otherwise.
template <class Set, class F>
int32_t mz_dispatch(mzgpu_ctx* ctx, int value, const char* what, F&& f) {
  return mz_dispatch_in(Set(), ctx, value, what, Set::kind, f);
}

// Row widths of the accumulable reduce with lane class C (1, 2, 4 or 8 lanes): the arrangement
// row (RowT above) and the output row (key, C x (count, sum_lo, sum_hi), flags, time, diff, pad).
// C = 1 is mzgpu_racc / mzgpu_rout.  The output widths skip 80 and 128 and 224 (see above).
template <int C>
struct LaneRows {
  static constexpr int ARR_NW = C == 1 ? 10 : (C == 2 ? 16 : (C == 4 ? 28 : 52));
  static constexpr int OUT_NW = C == 1 ? 8 : (C == 2 ? 12 : (C == 4 ? 18 : 30));
  static constexpr int OUT_TW = 3 * C + 2;  // time word of an output row (the diff follows)
};
static inline int mz_lane_class(uint32_t n_lanes) { return n_lanes <= 1 ? 1 : (n_lanes <= 2 ? 2 : (n_lanes <= 4 ? 4 : 8)); }
static inline int mz_lane_arr_bytes(int c) { return c == 1 ? 80 : (c == 2 ? 128 : (c == 4 ? 224 : 416)); }
static inline int mz_lane_out_bytes(int c) { return c == 1 ? 64 : (c == 2 ? 96 : (c == 4 ? 144 : 240)); }

// Monotonic MIN / MAX reduce (mzgpu_reduce_monotonic_new) with lane class C (4: 1-4 lanes, 8: 5-8
// lanes): the arrangement row (RowT<48> / RowT<112>) and the output row (key, C values, time, diff).
template <int C>
struct MonoRows {
  static constexpr int ARR_NW = C == 4 ? 6 : 14;
  static constexpr int OUT_NW = C + 3;
};
struct MonoClasses : IntSet<4, 8> {
  static constexpr const char* kind = "monotonic lane class";
};
static inline int mz_mono_class(uint32_t n_lanes) { return n_lanes <= 4 ? 4 : 8; }
static inline int mz_mono_arr_bytes(int c) { return c == 4 ? 48 : 112; }
static inline int mz_mono_out_bytes(int c) { return c == 4 ? 56 : 88; }

// Semigroup::plus_equals on the diff words, by the row's semigroup SG.
// MZ_SG_SUM: ND >= 8 is the accumulable diff: word 0 is the
// total, lane l spans words 1+6l .. 6+6l, and its words 1,2 (acc_lo, acc_hi) form an i128
// (src/compute/src/render/reduce.rs:1940-2041).  ND == 8 is one lane plus a pad word.
// MZ_SG_MAX: the monotonic reduce's Vec<ReductionMonoid> (reduce.rs:2193-2233), every lane
// encoded as an unsigned max (MonoRows): per-word max, zero the identity.
template <int ND, int SG = MZ_SG_SUM>
__host__ __device__ __forceinline__ void diff_add(u64* a, const u64* b) {
  if (SG == MZ_SG_MAX) {
#pragma unroll
    for (int w = 0; w < ND; ++w) a[w] = b[w] > a[w] ? b[w] : a[w];
  } else if (ND >= 8) {
    a[0] += b[0];
#pragma unroll
    for (int l = 0; l < (ND - 1) / 6; ++l) {
      u64* x = a + 1 + 6 * l;
      const u64* y = b + 1 + 6 * l;
      x[0] += y[0];
      u64 lo = x[1] + y[1];
      u64 carry = lo < x[1] ? 1 : 0;
      x[1] = lo;
      x[2] = x[2] + y[2] + carry;
      x[3] += y[3];
      x[4] += y[4];
      x[5] += y[5];
    }
  } else {
    a[0] += b[0];  // ND == 2 is (diff, pad): pad stays 0
  }
}
// IsZero: MZ_SG_MAX is never zero (reduce.rs:2235-2244), so a key stays once a row was accepted
template <int ND, int SG = MZ_SG_SUM>
__host__ __device__ __forceinline__ bool diff_is_zero(const u64* a) {
  if (SG == MZ_SG_MAX) return false;
  if (ND == 8) return (a[0] | a[1] | a[2] | a[3] | a[4] | a[5] | a[6]) == 0;
  if (ND > 8) {
    u64 x = 0;
#pragma unroll
    for (int w = 0; w < ND; ++w) x |= a[w];  // pad words stay zero
    return x == 0;
  }
  return a[0] == 0;
}
#ifdef __CUDACC__
// diff_add into global or shared memory by atomics, for the multi-lane diffs (ND > 8); the
// atomic that wraps a lane's acc_lo carries into its acc_hi
template <int ND>
__device__ __forceinline__ void atomic_lanes_add(u64* __restrict__ acc, const u64* d) {
  if (d[0]) atomicAdd((unsigned long long*)&acc[0], (unsigned long long)d[0]);
#pragma unroll
  for (int l = 0; l < (ND - 1) / 6; ++l) {
    u64* x = acc + 1 + 6 * l;
    const u64* y = d + 1 + 6 * l;
    if (y[0]) atomicAdd((unsigned long long*)&x[0], (unsigned long long)y[0]);
    const u64 old = atomicAdd((unsigned long long*)&x[1], (unsigned long long)y[1]);
    const u64 hi = y[2] + ((old + y[1]) < old ? 1 : 0);
    if (hi) atomicAdd((unsigned long long*)&x[2], (unsigned long long)hi);
    if (y[3]) atomicAdd((unsigned long long*)&x[3], (unsigned long long)y[3]);
    if (y[4]) atomicAdd((unsigned long long*)&x[4], (unsigned long long)y[4]);
    if (y[5]) atomicAdd((unsigned long long*)&x[5], (unsigned long long)y[5]);
  }
}
// diff_add of MZ_SG_MAX rows by atomics (zero-initialised accumulators: zero is the identity)
template <int ND>
__device__ __forceinline__ void atomic_diff_max(u64* __restrict__ acc, const u64* d) {
#pragma unroll
  for (int w = 0; w < ND; ++w)
    if (d[w]) atomicMax((unsigned long long*)&acc[w], (unsigned long long)d[w]);
}
#endif

// ----------------------------------------------------------- device helpers
#ifdef __CUDACC__
__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ u32 warp_id() { return threadIdx.x >> 5; }

// Block-wide exclusive scan of one u32 per thread (blockDim.x <= 1024, multiple
// of 32).  Returns the exclusive prefix; *total receives the block sum.
// `smem` must hold 33 u32.
__device__ __forceinline__ u32 block_exclusive_scan(u32 v, u32* smem, u32* total) {
  u32 lane = lane_id(), warp = warp_id();
  u32 incl = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    u32 o = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= (u32)off) incl += o;
  }
  if (lane == 31) smem[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    u32 nw = (blockDim.x + 31) >> 5;
    u32 w = lane < nw ? smem[lane] : 0;
    u32 wi = w;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      u32 o = __shfl_up_sync(0xffffffffu, wi, off);
      if (lane >= (u32)off) wi += o;
    }
    smem[lane] = wi - w;  // exclusive warp offsets
    if (lane == 31) smem[32] = wi;
  }
  __syncthreads();
  u32 res = smem[warp] + incl - v;
  *total = smem[32];
  __syncthreads();
  return res;
}

__device__ __forceinline__ u64 dlen_get(const DLen& l) { return l.p != nullptr ? *l.p : l.imm; }

// ---- chained scan across tiles (decoupled look-back), 64-bit totals.
// State word: [epoch:20][status:2][value:42].  A stale word (older epoch) reads
// as "not published", so the state array never needs clearing between launches.
constexpr u64 LB_VALUE_MASK = (1ull << 42) - 1;
constexpr u64 LB_PARTIAL = 1, LB_INCLUSIVE = 2;
__device__ __forceinline__ u64 lb_pack(u32 epoch, u64 status, u64 value) {
  return ((u64)epoch << 44) | (status << 42) | (value & LB_VALUE_MASK);
}
// Next tile for this CTA (tiles are handed out in order, so every predecessor
// of a tile has started: the look-back cannot deadlock).  All threads call it.
__device__ __forceinline__ u32 lb_next_tile(const LookBack& lb, u32* s_tile) {
  __syncthreads();
  if (threadIdx.x == 0) *s_tile = atomicAdd(lb.ticket, 1u);
  __syncthreads();
  return *s_tile;
}
// Exclusive prefix of `total` over all tiles before `tile`; publishes this
// tile's inclusive prefix.  Called by every thread of the CTA (warp 0 works);
// `s_bcast` is one shared u64.
__device__ __forceinline__ u64 lb_exclusive_prefix(const LookBack& lb, u32 tile, u64 total, u64* s_bcast) {
  if (threadIdx.x < 32) {
    const u32 lane = threadIdx.x;
    volatile u64* st = lb.state;
    u64 excl = 0;
    if (tile == 0) {
      if (lane == 0) st[0] = lb_pack(lb.epoch, LB_INCLUSIVE, total);
    } else {
      if (lane == 0) st[tile] = lb_pack(lb.epoch, LB_PARTIAL, total);
      // Each lane reads LBW consecutive predecessors per round (independent loads), so one round
      // covers 32 * LBW tiles: an update batch's few hundred tiles all start together, and the
      // walk would otherwise pay one memory round trip per 32 of them.
      constexpr int LBW = 4;
      long long hi = (long long)tile - 1;  // nearest unread predecessor
      while (true) {
        u64 w[LBW];
#pragma unroll
        for (int j = 0; j < LBW; ++j) {
          const long long idx = hi - (long long)(lane * LBW + j);
          w[j] = idx >= 0 ? st[idx] : 0;
        }
        int fj = LBW;  // this lane's nearest inclusive predecessor
        u64 contrib = 0;
#pragma unroll
        for (int j = 0; j < LBW; ++j) {
          const long long idx = hi - (long long)(lane * LBW + j);
          if (fj == LBW) {
            if (idx < 0) {
              fj = j;  // before tile 0: an inclusive zero
            } else {
              u64 x = w[j];
              u64 status = ((u32)(x >> 44) == lb.epoch) ? ((x >> 42) & 3) : 0;
              while (status == 0) {
                x = st[idx];
                status = ((u32)(x >> 44) == lb.epoch) ? ((x >> 42) & 3) : 0;
              }
              contrib += x & LB_VALUE_MASK;
              if (status == LB_INCLUSIVE) fj = j;
            }
          }
        }
        const u32 incl_mask = __ballot_sync(0xffffffffu, fj < LBW);
        const u32 first = __ffs(incl_mask) - 1;
        if (incl_mask != 0 && lane > first) contrib = 0;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, off);
        excl += contrib;
        if (incl_mask != 0) break;
        hi -= 32 * LBW;
      }
      if (lane == 0) st[tile] = lb_pack(lb.epoch, LB_INCLUSIVE, excl + total);
    }
    if (lane == 0) *s_bcast = excl;
  }
  __syncthreads();
  const u64 r = *s_bcast;
  __syncthreads();
  return r;
}

// Single-block exclusive scan of per-tile counts, in place; the grand total is
// written to *total_out.  n_tiles is small (n / 512), so one CTA suffices.
static __global__ void __launch_bounds__(1024) k_scan_tiles(u32* __restrict__ counts, u64 n_tiles,
                                                            u64* __restrict__ total_out) {
  __shared__ u32 sm[34];
  u32 carry = 0;
  for (u64 base = 0; base < n_tiles; base += 1024) {
    u64 i = base + threadIdx.x;
    u32 v = i < n_tiles ? counts[i] : 0;
    u32 total;
    u32 ex = block_exclusive_scan(v, sm, &total);
    if (i < n_tiles) counts[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) *total_out = carry;
}

// 128-bit vectorised global loads/stores of row words (rows are 16-byte aligned
// for every row width we use: 16, 32, 48, 64, 80).
template <int NW>
__device__ __forceinline__ void load_row(const u64* __restrict__ base, u64 idx, u64* r) {
  const u64* p = base + idx * NW;
  if (NW % 2 == 0) {
#pragma unroll
    for (int i = 0; i < NW; i += 2) {
      ulonglong2 v = *reinterpret_cast<const ulonglong2*>(p + i);
      r[i] = v.x;
      r[i + 1] = v.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < NW; ++i) r[i] = p[i];
  }
}
template <int NW>
__device__ __forceinline__ void store_row(u64* __restrict__ base, u64 idx, const u64* r) {
  u64* p = base + idx * NW;
  if (NW % 2 == 0) {
#pragma unroll
    for (int i = 0; i < NW; i += 2) {
      ulonglong2 v;
      v.x = r[i];
      v.y = r[i + 1];
      *reinterpret_cast<ulonglong2*>(p + i) = v;
    }
  } else {
#pragma unroll
    for (int i = 0; i < NW; ++i) p[i] = r[i];
  }
}

// 64-bit mixer for the open-addressing hash index (murmur3 finalizer).
__host__ __device__ __forceinline__ u64 mix64(u64 k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}

// Closure evaluation on device: same descriptor semantics as include/mzgpu.h.
__host__ __device__ __forceinline__ u64 field_get(const mzgpu_field& f, u64 key, u64 v1, u64 v2) {
  u64 w = f.src == MZGPU_SRC_KEY ? key : (f.src == MZGPU_SRC_VAL1 ? v1 : v2);
  w >>= f.shift;
  if (f.bits < 64) w &= ((u64)1 << f.bits) - 1;
  return w;
}
__host__ __device__ __forceinline__ bool closure_eval(const mzgpu_closure& c, u64 key, u64 v1, u64 v2,
                                                      u64* okey, u64* oval) {
  for (u32 i = 0; i < c.n_filters; ++i) {
    const mzgpu_filter& f = c.filters[i];
    u64 x = field_get(f.field, key, v1, v2);
    bool ok;
    switch (f.op) {
      case MZGPU_CMP_EQ: ok = x == f.rhs; break;
      case MZGPU_CMP_NE: ok = x != f.rhs; break;
      case MZGPU_CMP_LT: ok = x < f.rhs; break;
      case MZGPU_CMP_LE: ok = x <= f.rhs; break;
      case MZGPU_CMP_GT: ok = x > f.rhs; break;
      default: ok = x >= f.rhs; break;
    }
    if (!ok) return false;
  }
  u64 k = 0, v = 0;
  for (u32 i = 0; i < c.n_key_fields; ++i)
    k |= field_get(c.key_fields[i], key, v1, v2) << c.key_fields[i].dst_shift;
  if (c.expr_kind == MZGPU_EXPR_MUL_CONST_MINUS) {
    u64 a = field_get(c.expr_a, key, v1, v2);
    u64 b = field_get(c.expr_b, key, v1, v2);
    v = a * (c.expr_c - b);
  } else {
    for (u32 i = 0; i < c.n_val_fields; ++i)
      v |= field_get(c.val_fields[i], key, v1, v2) << c.val_fields[i].dst_shift;
  }
  *okey = k;
  *oval = v;
  return true;
}
#endif  // __CUDACC__

// ------------------------------------------------------- kernel entry points
// (implemented in the .cu files; all asynchronous on ctx->stream unless noted)

// sort.cu: stable LSD radix sort of a permutation by the key words of `rows`.
// On return d_perm (u32[n]) holds the sorted order.  Synchronises once to read
// the key ranges.
int32_t mz_sort_perm(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, DevMem* perm_out);

// consolidate.cu
// rows[perm] gathered into a dense sorted array
int32_t mz_gather_rows(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, const u32* d_perm, u64 n,
                       void* d_out);
// Sum diffs of equal neighbours in a sorted array and drop zeros.  Output is
// written to d_out (capacity n rows); *n_out is read back (one sync).
int32_t mz_consolidate_sorted(mzgpu_ctx* ctx, int row_bytes, const void* d_sorted, u64 n,
                              void* d_out, u64* n_out);
// sort + gather + consolidate; output array is allocated (capacity n rows).
int32_t mz_sort_consolidate(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, DevMem* out,
                            u64* n_out);

// fused.cu: consolidate(A ++ B with times advanced to `since`), split by `upper`,
// hash index — ONE cooperative kernel, no host read-back.  Inputs larger than
// MZ_FUSED_MAX_ROWS take the multi-kernel path (sort.cu, consolidate.cu, ...).
struct FusedJob {
  int rb = 0;
  const void* a = nullptr;  // first input (for a merge: the older batch)
  const void* b = nullptr;  // optional second input
  DLen na = {nullptr, 0}, nb = {nullptr, 0};
  u64 cap = 0;                          // host upper bound on na + nb (sizes every buffer)
  u64 since = 0;                        // advance_by(since)
  u64 upper = MZGPU_FRONTIER_EMPTY;     // rows with time < upper go to `rows`, the rest to `keep`
  bool want_index = false;
  bool merge = false;  // a and b are each sorted and consolidated (a batch merge): merge path, no sort
};
struct FusedOut {
  DevMem rows;  // consolidated (shipped) rows, capacity rows_cap
  u64 rows_cap = 0;
  DevMem table;  // hash index, if requested
  DevMem keep;   // rows with time >= upper (allocated only when upper is a real frontier)
  Lazy4 st;      // [0] rows out, [1] table mask, [2] distinct keys, [3] longest key run (saturates at 1024)
  Lazy4 kst;     // [0] rows kept, [1] min kept time (~0 if none), [2] max input time
};
int32_t mz_fused_consolidate(mzgpu_ctx* ctx, const FusedJob& job, FusedOut* out);
// k independent jobs of one row width in one cooperative launch (k <= MZ_FUSED_MANY_MAX)
#define MZ_FUSED_MANY_MAX 4
int32_t mz_fused_consolidate_many(mzgpu_ctx* ctx, int k, const FusedJob* jobs, FusedOut* outs);
// mergepath.cu: two sorted, consolidated R32 arrays merged (times advanced to `since`), consolidated and
// indexed by three ordinary stream-ordered launches; results as the fused kernel's merge leaves them
int32_t mz_merge_r32_async(mzgpu_ctx* ctx, const void* d_a, DLen na, const void* d_b, DLen nb, u64 cap, u64 since,
                           FusedOut* res);
// prepare now, launch with the other deferred jobs at mz_fused_flush (host.cu: mz_flush_deferred)
int32_t mz_fused_defer(mzgpu_ctx* ctx, const FusedJob& job, FusedOut* out);
int32_t mz_fused_flush(mzgpu_ctx* ctx);
void mz_fused_deferred_free(mzgpu_ctx* ctx);
size_t mz_fused_ctl_bytes();
#define MZ_FUSED_MAX_ROWS (2u << 20)
// ... judged by the exact row count when the host knows it.  When it only has an
// upper bound (the count is still on the device), the fused kernel takes
// capacities up to MZ_FUSED_MAX_CAP: buffers are sized by the bound, work by the
// actual count, and a loose bound is the common case (probe fan-out bounds).
#define MZ_FUSED_MAX_CAP (32u << 20)
static inline bool mz_use_fused(bool exact, u64 ub) {
  return exact ? ub <= MZ_FUSED_MAX_ROWS : ub <= MZ_FUSED_MAX_CAP;
}

// merge.cu: merge two sorted consolidated arrays; times are advanced to
// max(time, since) on the way; result is consolidated.
int32_t mz_merge_consolidate(mzgpu_ctx* ctx, int row_bytes, const void* d_a, u64 na, const void* d_b,
                             u64 nb, u64 since, DevMem* out, u64* n_out);
// stable partition of sorted rows by time < upper: ship (t < upper) and keep.
int32_t mz_extract(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, u64 upper, DevMem* ship,
                   u64* n_ship, DevMem* keep, u64* n_keep, u64* min_keep_time);

// index.cu: open-addressing hash index over the distinct keys of a sorted array.
struct HashSlot {
  u64 key;
  u64 meta;  // 0 = empty; bits [0,44): first row index + 1; bits [44,64): the key's run
             // length if the builder knows it (else 0: the reader scans until the key changes)
};
#define MZ_SLOT_ROW_MASK ((1ull << 44) - 1)
#define MZ_SLOT_LEN_MAX 0xfffffull
int32_t mz_count_keys(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, u64* n_keys, u64* max_run);
int32_t mz_build_index(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, u64 n_keys,
                       DevMem* table, u64* table_slots);

int32_t mz_seek_keys(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, DLen n, const u64* d_probe, u64 n_probe,
                     u64* d_out);
int32_t mz_key_page(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n_rows, u64 first_ordinal, u64 max_keys,
                    u64* d_out);

// probe.cu
struct BatchView {  // device-visible description of one batch of a trace
  const u64* rows;
  const HashSlot* table;
  u64 n;
  u64 mask;        // table_slots - 1
  const u64* hdr;  // if set, n = hdr[0] and mask = hdr[1] live in device memory (batch built
                   // by a kernel still in flight; see Lazy4)
};
#ifdef __CUDACC__
__device__ __forceinline__ u64 bv_n(const BatchView& b) { return b.hdr != nullptr ? b.hdr[0] : b.n; }
__device__ __forceinline__ u64 bv_mask(const BatchView& b) { return b.hdr != nullptr ? b.hdr[1] : b.mask; }
#endif
#define MZ_MAX_TRACE_BATCHES 64
struct TraceView {
  BatchView b[MZ_MAX_TRACE_BATCHES];
  u32 n_batches;
};
#define MZ_PROBE_HALF_LE 0
#define MZ_PROBE_HALF_LT 1
#define MZ_PROBE_JOIN 2  // join_core: no time filter, time = max(t1, t2, meet)
struct ProbeParams {
  int mode;
  u64 meet;         // join_core capability time
  int has_closure;  // 0: identity -> R40 (key, v1, v2)
  int swap_vals;    // join_core side 1: probe rows are val2, lookup rows are val1
  mzgpu_closure closure;
};
// An MfpPlan closure on a probe (mzgpu_join_closure): the plan in device memory and the output row width.  The
// single-pass forms write the R32 error rows at errs[(*err_len)++] (err_cap rows; *err_len zeroed by the caller);
// the two-pass form allocates them.
struct MfpDevPlan;
struct MfpProbe {
  const MfpDevPlan* pl;
  int out_rb;
  u64* errs;
  u64 err_cap;
  u64* err_len;
};
#define MZ_PROBE_MANY_MAX 3
struct ProbeJobHost {
  const u64* d_stream;
  DLen n;
  u64 n_ub;
  const TraceView* trace;
  const ProbeParams* pp;
  int chain;  // jobs with equal chain ids are consecutive and append to one output
  bool has_pre = false;                 // map in front of the probe: drop rows at skip_time, apply `pre`
  const mzgpu_closure* pre = nullptr;   // (nullptr: identity)
  u64 skip_time = MZGPU_FRONTIER_EMPTY;
  u64* d_out;
  DLen out_base;
  u64 out_cap;
  u64* d_out_len;
  const MfpProbe* mfp = nullptr;  // an MfpPlan closure instead of pp's (every job of a launch, or none)
};
int32_t mz_probe_async_many(mzgpu_ctx* ctx, int k, const ProbeJobHost* jobs);
// tiles the single-pass probe cuts `n_ub` probe rows into (rows per tile shrink with the trace's
// batch count so that a tile's hit list fits in shared memory)
static inline u64 mz_probe_tile_rows(u64 n_ub, u32 n_batches) {
  // 8 warps per tile, each with a private hit list of 256 entries: rows per warp x batches <= 256
  (void)n_ub;
  const u64 per_warp = n_batches <= 8 ? 32u : (n_batches <= 16 ? 16u : (n_batches <= 32 ? 8u : 4u));
  return 8 * per_warp;
}
static inline u64 mz_probe_tiles(u64 n_ub, u32 n_batches) {
  const u64 tr = mz_probe_tile_rows(n_ub, n_batches);
  return (n_ub + tr - 1) / tr;
}
// Probe `n` R32 stream rows against the trace; appends results to d_out
// (allocated here) and returns the count.  One sync (to size the output).
// With an MfpPlan closure (`mfp`) the error rows go to `errs` (allocated here), *n_errs of them.
int32_t mz_probe(mzgpu_ctx* ctx, const u64* d_stream, u64 n, const TraceView& trace,
                 const ProbeParams& pp, DevMem* out, u64* n_out, const MfpProbe* mfp = nullptr,
                 DevMem* errs = nullptr, u64* n_errs = nullptr);
// Single-pass form: `n` is read on the device, results are written at
// d_out[out_base ...] (capacity out_cap rows: the caller guarantees it with a
// bound, ctx->d_status records a violation) and the new length is left in
// *d_out_len.  No host round trip.
int32_t mz_probe_async(mzgpu_ctx* ctx, const u64* d_stream, DLen n, u64 n_ub, const TraceView& trace,
                       const ProbeParams& pp, u64* d_out, DLen out_base, u64 out_cap, u64* d_out_len,
                       const MfpProbe* mfp = nullptr);
int32_t mz_map_rows_async(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const mzgpu_closure* closure,
                          u64 skip_time, u64* d_out, DLen out_base, u64 out_cap, u64* d_out_len);
// Apply a closure to R32 rows (val2 = 0); optional skip of rows at `skip_time`.
int32_t mz_map_rows_dev(mzgpu_ctx* ctx, const u64* d_rows, u64 n, const mzgpu_closure* closure,
                        u64 skip_time, DevMem* out, u64* n_out);

// reduce.cu
int32_t mz_explode(mzgpu_ctx* ctx, const u64* d_r32, DLen n, u64 n_ub, int agg_kind, u64* d_racc);
// the lanes operator's explode_one: R32 / R40 rows -> one arrangement row of class C each
struct LaneSet {
  mzgpu_accum_lane lane[MZGPU_MAX_ACCUM_LANES];
  u32 n;         // lanes in use; the class's other lanes stay zero
  u32 in_words;  // 4 (R32) or 5 (R40)
  u32 f64_mask;  // bit l: lane l is MZGPU_AGG_COUNT_SUM_F64
  u32 distinct_mask;  // bit l: lane l carries MZGPU_ACCUM_DISTINCT (its words stay zero in the explode)
};
int32_t mz_explode_lanes(mzgpu_ctx* ctx, int c, const u64* d_rows, DLen n, u64 n_ub, const LaneSet& ls,
                         u64* d_arr);
// the distinct lanes' pair rows: for the j-th set bit l of ls.distinct_mask, d_pairs[j] receives the R32
// rows (key, lane l's value, time, diff) of the input, and *d_lens[j] the row count unless d_lens[j] is
// nullptr (one launch)
int32_t mz_distinct_pairs(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const LaneSet& ls,
                          u64* const* d_pairs, u64* const* d_lens);
// Presence changes of the distinct lanes' new pair batches (one launch per MZ_LB_TILES tiles): one class-c
// arrangement row per change of a (key, value) pair between zero and non-zero accumulated multiplicity,
// appended at d_out (capacity out_cap rows, at least the pair batches' total length); the row count is
// left in len->v[*len_word] on the device.
struct DistinctJobHost {
  const u64* rows;  // the new pair batch (R32, sorted and consolidated)
  DLen n;
  u64 n_ub;
  u32 lane;               // lane index in the class row
  const TraceView* prior;  // the pair arrangement's earlier batches
};
int32_t mz_distinct_presence(mzgpu_ctx* ctx, int c, int k, const DistinctJobHost* jobs, u64* d_out, u64 out_cap,
                             Lazy4* len, int* len_word);
struct TopKParams {
  i64 limit;  // < 0: none
  u64 offset;
  int descending;
};
int32_t mz_reduce_minmax_async(mzgpu_ctx* ctx, const u64* d_batch_rows, DLen n, u64 n_ub,
                               const TraceView& prior, int agg_kind, const TopKParams& tp, u64* d_out,
                               u64 out_cap, u64* d_out_len);
// `c` is the lane class (1 for every mzgpu_reduce_new kind); for c >= 2 the lanes' kinds come
// from `ls` (f64_mask, n) and agg_kind is unused.  `hv`: the lanes operator's HAVING program
// (validated, at least one predicate), run by the filtered kernels; nullptr runs the unfiltered ones.
int32_t mz_reduce_corrections_async(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, DLen n, u64 n_ub,
                                    const TraceView& prior, int agg_kind, const LaneSet* ls, u64* d_out,
                                    u64 out_cap, u64* d_out_len, const mzgpu_having* hv = nullptr);
int32_t mz_reduce_corrections(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, u64 n, const TraceView& prior,
                              int agg_kind, const LaneSet* ls, DevMem* out, u64* n_out,
                              const mzgpu_having* hv = nullptr);
// the monotonic MIN / MAX reduce (mzgpu_reduce_monotonic_new): lane l's arrangement word is its value ^ xm[l]
// (2^63 for a signed lane, then all ones for MIN), so every lane accumulates as an unsigned max
struct MonoXor {
  u64 xm[MZGPU_MAX_ACCUM_LANES];
  u32 n;  // lanes in use; the class's other lanes stay zero
};
// rows with diff > 0 -> class-c arrangement rows at d_arr, every other row -> an R16 (time, +1) row at
// d_errs; their counts are left in d_cnt[0] and d_cnt[1] (two words of a counter block, zeroed here)
int32_t mz_monotonic_explode(mzgpu_ctx* ctx, int c, const u64* d_rows, DLen n, u64 n_ub, const LaneSet& ls,
                             const MonoXor& mx, u64* d_arr, u64* d_errs, u64* d_cnt);
// the R32 / R40 rows with value word 1 masked by m1 and word 2 (R40) by m2
int32_t mz_monotonic_mask(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, u32 in_words, u64 m1, u64 m2,
                          u64* d_out);
int32_t mz_monotonic_corrections_async(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, DLen n, u64 n_ub,
                                       const TraceView& prior, const MonoXor& mx, u64* d_out, u64 out_cap,
                                       u64* d_out_len);
int32_t mz_monotonic_corrections(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, u64 n, const TraceView& prior,
                                 const MonoXor& mx, DevMem* out, u64* n_out);
// the hierarchical MIN / MAX reduce (mzgpu_reduce_hierarchical_new): corrections of a sealed batch of masked
// input rows (ls.in_words words) against the prior arrangement, rows of the monotonic output width of class c
// (consolidated), and R32 error rows (key, 0, time, +-1; unordered) at d_errs[*d_err_len++] (the counter is
// zeroed here).  Single pass: out_cap = 2 * n_ub and err_cap = n_ub always suffice.
int32_t mz_hier_corrections_async(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, DLen n, u64 n_ub,
                                  const TraceView& prior, const LaneSet& ls, const MonoXor& mx, u64* d_out,
                                  u64 out_cap, u64* d_out_len, u64* d_errs, u64 err_cap, u64* d_err_len);
// the two-pass form (count, read back, write) for a batch past the single-pass bound; err_cap = n suffices
int32_t mz_hier_corrections(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, u64 n, const TraceView& prior,
                            const LaneSet& ls, const MonoXor& mx, DevMem* out, u64* n_out, u64* d_errs, u64 err_cap,
                            u64* d_err_len);
// the monotonic TopK (mzgpu_topk_monotonic_new): order word j of a row = field_get(lane j) (sign-extended when
// signed) ^ xm[j] (2^63 for a signed lane, then all ones for a descending one); lanes n..2 stay zero
struct TopKOrder {
  mzgpu_field f[3];
  u32 sign_extend[3];
  u64 xm[3];
  u32 n;
  u32 in_words;  // 4 (R32) or 5 (R40)
  i64 limit;     // >= 0; INT64_MAX is LIMIT NULL
};
// rows with diff > 0 -> 72-byte window rows at d_arr, every other row -> an R16 (time, +1) row at d_errs;
// their counts are left in d_cnt[0] and d_cnt[1] (two words of a counter block, zeroed here)
int32_t mz_topk_explode(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const TopKOrder& to, u64* d_arr,
                        u64* d_errs, u64* d_cnt);
// The window changes of the new 72-byte rows (sorted, consolidated) against the window arrangement `prior`:
// 72-byte rows at d_win and the same rows at the input width at d_out (each key's sorted), out_cap rows each.
int32_t mz_topk_window_async(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const TraceView& prior,
                             const TopKOrder& to, u64* d_win, u64* d_out, u64 out_cap, u64* d_out_len);
int32_t mz_topk_window(mzgpu_ctx* ctx, const u64* d_rows, u64 n, const TraceView& prior, const TopKOrder& to,
                       DevMem* win, DevMem* out, u64* n_out);
// the basic TopK (mzgpu_topk_basic_new): every input row -> one 72-byte row (row i at d_arr[i])
int32_t mz_topk_basic_explode(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const TopKOrder& to, u64* d_arr);
// The changes of the new 72-byte rows (sorted, consolidated, any diff) against the input arrangement `prior` and
// the negatives arrangement `negs_tv` (R32): window changes at the input width at d_out (consolidated), R32 error
// rows (key, 0, time, +-1) at d_errs[d_side_len[0]++] and R32 negatives deltas (key, 0, time, delta) at
// d_negs[d_side_len[1]++], both unordered (the two counters are zeroed here).  side_cap = the new row count
// suffices (at most one of each per key and new time).  Single pass: out_cap = 2 * limit per new row suffices.
int32_t mz_topk_basic_async(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const TraceView& prior,
                            const TraceView& negs_tv, const TopKOrder& to, i64 offset, u64* d_out, u64 out_cap,
                            u64* d_out_len, u64* d_errs, u64* d_negs, u64 side_cap, u64* d_side_len);
// the two-pass form (count, read back, write): past the single-pass bound, and for LIMIT NULL
int32_t mz_topk_basic(mzgpu_ctx* ctx, const u64* d_rows, u64 n, const TraceView& prior, const TraceView& negs_tv,
                      const TopKOrder& to, i64 offset, DevMem* out, u64* n_out, u64* d_errs, u64* d_negs,
                      u64 side_cap, u64* d_side_len);

// correction.cu (time-major rows: (time, key, val | diff))
// column.cu (columnar wire format, f4)
int32_t mz_col_decode_fixed(mzgpu_ctx* ctx, int nw, const u64* d_words, u64 n, const u64* off_words, u64* d_dst,
                            u64 base);
int32_t mz_col_encode_fixed(mzgpu_ctx* ctx, int nw, const u64* d_rows, u64 first, u64 n, const u64* off_words,
                            u64* d_words);
int32_t mz_col_decode_rows(mzgpu_ctx* ctx, const u64* d_words, u64 n, const u64* off_words, u64 key_bytes,
                           u64 val_bytes, u64* d_dst, u64 base, u64* d_flag);
int32_t mz_col_row_prefix(mzgpu_ctx* ctx, const u64* d_rows, u64 first, u64 n, u64* d_bsum, u64* d_pk, u64* d_pv,
                          u64* d_tot);
int32_t mz_col_encode_rows(mzgpu_ctx* ctx, const u64* d_rows, u64 first, u64 s, u64 n, const u64* d_pk,
                           const u64* d_pv, const u64* off_words, u64* d_words);
int32_t mz_col_cuts(mzgpu_ctx* ctx, const u64* d_pk, const u64* d_pv, u64 n, u64* d_cuts, u64 cap, u64* d_n_cuts);
int32_t mz_corr_to_td(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, u64 since, bool negate, u64* d_td, DLen base,
                      u64 cap_rows, u64* d_out_len);
int32_t mz_corr_advance(mzgpu_ctx* ctx, u64* d_td, DLen n, u64 n_ub, u64 since);
int32_t mz_corr_split(mzgpu_ctx* ctx, const u64* d_td, DLen n, u64 upper, u64* d_out);
int32_t mz_corr_from_td(mzgpu_ctx* ctx, const u64* d_td, DLen n, u64 n_ub, u64* d_dst, DLen base, u64 cap_rows,
                        u64* d_out_len);

// exchange.cu
#define MZ_MAX_EXCHANGE 8
#define MZ_P2P_MAX_PEERS 16
#define MZ_P2P_HEADER_BYTES 4096
size_t mz_p2p_zone_bytes(u64 landing_rows, u32 region_rb, u32 peers);
int32_t mz_p2p_send(mzgpu_ctx* ctx, u32 k, const int* row_bytes, const void* const* d_rows, const DLen* n,
                    const u64* n_ub);
int32_t mz_p2p_recv(mzgpu_ctx* ctx, u32 k, const int* row_bytes, void* const* d_out, const u64* out_cap,
                    u64* const* d_out_len);
int32_t mz_partition_many(mzgpu_ctx* ctx, u32 k, const int* row_bytes, const void* const* d_rows, const DLen* n,
                          const u64* n_ub, u32 peers, void* const* d_out, u64* d_counts, u64* d_cursors,
                          u64* d_send_by_peer /* [peer][k] */);
int32_t mz_partition(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, DLen n, u64 n_ub, u32 peers, void* d_out,
                     u64* d_counts /* 64 words */, u64* d_cursors /* 64 words */);

// mfp.cu: the temporal filter (mzgpu_mfp_new).  A plan as the kernels read it: the caller's descriptor plus
// the derived bound lists (program index in bits 0-2, bit 3: wrapped in step_mz_timestamp), in the order of
// MfpPlan::create_from; and the map expressions (mzgpu_mfp_new_map) with each predicate's support.
struct MfpDevPlan {
  mzgpu_mfp plan;
  u32 n_lower, n_upper;
  u32 lower[MZGPU_MFP_MAX_TEMPORAL], upper[MZGPU_MFP_MAX_TEMPORAL];
  i64 iv_us[MZGPU_MFP_MAX_CONSTS];  // interval constants folded to microseconds (MZGPU_HOP_TS_ADD_IV)
  mzgpu_mfp_map map;                // n_exprs == 0 without expressions
  i64 map_iv_us[MZGPU_MFP_MAX_CONSTS];
  u32 support[MZGPU_MFP_MAX_PREDICATES];  // expressions evaluated before predicate p
};
// k_mfp_eval takes the plan as a __grid_constant__ parameter beside 80 bytes of others: within the 4 KB of
// kernel parameters every CUDA 12 driver accepts
static_assert(sizeof(MfpDevPlan) + 80 <= 4096, "MfpDevPlan exceeds the kernel parameter limit");
// a segment: MZ_MFP_HDR header words (slice j's rows are [hdr[j], hdr[j + 1])), then the rows
#define MZ_MFP_HDR 72
#define MZ_MFP_MAX_SLOTS 65  // 64 bucket bounds and the overflow slot of an insert round
#define MZ_MFP_SLICES 32     // source slices per partition launch
struct MfpSlices {
  const u64* base[MZ_MFP_SLICES];
  u32 idx[MZ_MFP_SLICES];
  u32 n;
};
struct MfpBounds {
  u64 v[MZ_MFP_MAX_SLOTS];  // ascending; a row at time t goes to slot (# v <= t) - 1
  u32 nb;
};
int32_t mz_mfp_eval(mzgpu_ctx* ctx, const MfpDevPlan& pl, const u64* d_rows, DLen n, u64 n_ub, u64 upper, u64 until,
                    u64* ready, u64* held, u64* errs, u64* err_len);
// partition the rows of `chunks` into the nb slots of segment `dst`; `hist` and `cursor` are
// MZ_MFP_MAX_SLOTS words each, adjacent (cursor == hist + MZ_MFP_MAX_SLOTS); *total (if set) gets the row count
int32_t mz_mfp_partition(mzgpu_ctx* ctx, int rb, const MfpSlices* chunks, u32 n_chunks, u64 rows_ub,
                         const MfpBounds& b, u64* hist, u64* cursor, u64* dst, u64* total, u64* touched);
int32_t mz_mfp_min_time(mzgpu_ctx* ctx, int rb, const MfpSlices* chunks, u32 n_chunks, u64 rows_ub, u64* d_min);

// mfp.cu: FlatMap (mzgpu_flat_map_new).  The table function as the kernels read it beside the MfpPlan: its
// descriptor, its folded intervals, the timestamp step in microseconds and its number of arguments.
struct FlatMapDevPlan {
  MfpDevPlan mfp;
  mzgpu_table_func tf;
  i64 iv_us[MZGPU_MFP_MAX_CONSTS];
  i64 step_us;
  u32 n_args;
};
// k_fm_expand takes the plan as a __grid_constant__ parameter beside 96 bytes of others
static_assert(sizeof(FlatMapDevPlan) + 96 <= 4096, "FlatMapDevPlan exceeds the kernel parameter limit");
#define MZ_FM_TILE 1024  // input rows per tile of the count-and-scan kernel
// Per input row: the function's record (start, step, diff multiplier) and the inclusive 128-bit prefix of the
// function-row counts; the look-back state is 3 words per tile (flag, lo, hi), zeroed before the launch, with a
// tile ticket after it.  d_total gets (total lo, total hi, input rows).
struct FmRec {
  i64 start, step, mult;
};
int32_t mz_fm_count(mzgpu_ctx* ctx, const FlatMapDevPlan& pl, const u64* d_rows, DLen n, u64 n_ub, FmRec* rec,
                    ulonglong2* incl, u64* lb_state, u64* d_total, u64* errs, u64* err_len);
// one page: function rows [g, g + page) of the activation, through the MfpPlan into ready / held / errs
int32_t mz_fm_expand(mzgpu_ctx* ctx, const FlatMapDevPlan& pl, const u64* d_rows, const FmRec* rec,
                     const ulonglong2* incl, u64 n, unsigned __int128 g, u64 page, u64 upper, u64 until, u64* ready,
                     u64* held, u64* errs, u64* err_len);
// the least time of the input rows whose function rows are not all below ordinal g (atomicMin into *d_min)
int32_t mz_fm_min_time(mzgpu_ctx* ctx, int iw, const u64* d_rows, const ulonglong2* incl, u64 n,
                       unsigned __int128 g, u64* d_min);

// peek.cu: index peeks (mzgpu_peek_many).  A peek plan as the kernels read it: the MfpPlan over (key, val) and the
// finishing -- order lanes over the output words (encoded as TopKOrder does), the [offset, end) cut in units and the
// projection (identity when no word has fields).
struct PeekFin {
  mzgpu_field f[3];
  u32 sign_extend[3];
  u64 xm[3];
  u32 n_order;
  u32 out_words;  // 2 or 3
  u64 offset, end;  // end = offset + limit, saturating; UINT64_MAX without a limit
  u32 identity;
  u32 n_project[3];
  mzgpu_field project[3][MZGPU_MAX_FIELDS];
};
struct PeekDevPlan {
  MfpDevPlan mfp;
  PeekFin fin;
};
// A request as the kernels see it.  Gathered rows are R40 (slot, key, val, as_of, diff).  Slot i < k holds literal
// request i's pairs; slot k + j the ok trace at the j-th distinct as_of of the full scans, shared by every full-scan
// request at that as_of; slot err_base + j the error trace at the j-th distinct as_of.
#define MZ_PEEK_K 64
struct PeekScanJobs {  // the full scans of one trace: job j keeps rows with time <= as_of[j] as slot[j]
  u32 n;
  u32 slot[MZ_PEEK_K];
  u64 as_of[MZ_PEEK_K];
};
struct PeekLitSegs {  // literal keys [start[s], start[s + 1]) belong to slot[s] at as_of[s]
  u32 n;
  u64 start[MZ_PEEK_K + 1];
  u32 slot[MZ_PEEK_K];
  u64 as_of[MZ_PEEK_K];
};
struct PeekReqs {
  const PeekDevPlan* pl[MZ_PEEK_K];  // nullptr: the request is not run (decided on the host)
  u64 as_of[MZ_PEEK_K];
  u64 reqs[2 * MZ_PEEK_K];   // per ok slot (below err_base): the requests evaluated on its pairs, as a bit set
  int err_slot[MZ_PEEK_K];  // the request's error-trace slot, -1: no error trace
  u32 k;
  u32 err_base;
};
struct PeekDevResult {
  u64 kind;  // 0 or MZGPU_PEEK_ERR_*
  u64 n_rows;
  u64 lo;  // the request's rows are at staging byte offset lo * 40
  u64 d[4];
};
int32_t mz_peek_scan(mzgpu_ctx* ctx, const TraceView& tv, const PeekScanJobs& jobs, u64* d_out, u64 cap, u64* d_len);
int32_t mz_peek_lits(mzgpu_ctx* ctx, const u64* d_keys, const PeekLitSegs& segs, u64* d_rows);
int32_t mz_peek_unit(mzgpu_ctx* ctx, u64* d_rows, DLen n, u64 n_ub);
// pairs (consolidated R40 rows) -> 72-byte finishing rows (slot, o0, o1, o2, w0, w1, w2, copies, 0) at d_fin
// (count at *d_fin_len, zeroed by the caller), one per request of the pair's slot; failures as atomicMin of the row
// index into d_fail[request], an error-trace slot's first row into d_fail[slot]
int32_t mz_peek_eval(mzgpu_ctx* ctx, const u64* d_pairs, DLen n, u64 n_ub, u64 fin_cap, const PeekReqs& rq, u64* d_fin,
                     u64* d_fin_len, u64* d_fail);
// one block per request: its failure detail, or its cut and projected rows into d_stage
int32_t mz_peek_finish(mzgpu_ctx* ctx, const PeekReqs& rq, const u64* d_pairs, const u64* d_fail, const u64* d_fin,
                       DLen n_fin, u64* d_stage, PeekDevResult* d_res);

#ifdef __CUDACC__
// ---------------------------------------------------------- the MfpPlan interpreter (mfp.cu, probe.cu)
namespace {

// A stack value: v (an INT as i64, a BOOL as 0 / 1, an MZTS as u64 bits, a TS as i64 microseconds,
// a DATE as i64 days), err (0 or an MZGPU_*_ERR_* code, ordered as the EvalError variants) and the
// error payload.  No value is NULL (no nullable column is in the subset).  Types are host-checked
// (host.cu: validate_mfp_program), so the device only follows the opcodes.
struct MVal {
  u64 v;
  u32 err;
  u64 pay;
};

__device__ __forceinline__ u32 mfp_arith(u32 code, int w, i64 a, i64 b, i64* r) {
  const i64 lo = w == 32 ? (i64)(-2147483647 - 1) : (i64)0x8000000000000000ull;
  i64 x;
  bool ovf = false;
  if (code == MZGPU_HOP_ADD) {
    x = (i64)((u64)a + (u64)b);
    ovf = ((a ^ x) & (b ^ x)) < 0;
  } else if (code == MZGPU_HOP_SUB) {
    x = (i64)((u64)a - (u64)b);
    ovf = ((a ^ b) & (a ^ x)) < 0;
  } else if (code == MZGPU_HOP_MUL) {
    x = (i64)((u64)a * (u64)b);
    ovf = __mul64hi((long long)a, (long long)b) != (x >> 63);
  } else if (code == MZGPU_HOP_MOD) {  // checked_rem(b).unwrap_or(0): MIN % -1 is 0
    if (b == 0) return MZGPU_HAVING_ERR_DIVISION_BY_ZERO;
    x = b == -1 ? 0 : a % b;
  } else {
    if (b == 0) return MZGPU_HAVING_ERR_DIVISION_BY_ZERO;
    if (b == -1 && a == lo) return w == 32 ? MZGPU_HAVING_ERR_INT32_OUT_OF_RANGE : MZGPU_HAVING_ERR_INT64_OUT_OF_RANGE;
    x = a / b;
  }
  if (w == 32 && x != (i64)(int)x) ovf = true;
  if (ovf) return MZGPU_HAVING_ERR_NUMERIC_FIELD_OVERFLOW;
  *r = x;
  return 0;
}

// [LOW_DATE, HIGH_DATE + 1 day) in microseconds since 1970-01-01 (src/repr/src/adt/timestamp.rs:577-592)
constexpr i64 TS_LOW_US = -210863692800000000ll;
constexpr i64 TS_HIGH_US = 8210266876799999999ll;

__device__ __forceinline__ u64 mfp_field(const u64* w, const mzgpu_having_op& o) {
  u64 a = w[o.arg] >> o.shift;
  if (o.bits < 64) {
    a &= (1ull << o.bits) - 1;
    if (o.sign_extend && ((a >> (o.bits - 1)) & 1)) a |= ~0ull << o.bits;
  }
  return a;
}

// Runs one program over the input words w and the expression values mv (every one a MZGPU_HOP_MAP may read is
// evaluated, without error); its constants are consts / iv_us.  Returns the value left on the stack.
__device__ __noinline__ MVal mfp_run(const mzgpu_having_op* ops, u32 n_ops, const mzgpu_having_const* consts,
                                     const i64* iv_us, const u64* w, const u64* mv) {
  constexpr int D = MZGPU_HAVING_MAX_STACK;
  u64 v[D], pay[D];
  u32 err[D];
  int sp = 0;
  for (u32 i = 0; i < n_ops; ++i) {
    const mzgpu_having_op o = ops[i];
    const u32 code = o.code;
    if (code == MZGPU_HOP_COL || code == MZGPU_HOP_COL_MZTS || code == MZGPU_HOP_COL_TS ||
        code == MZGPU_HOP_COL_DATE || code == MZGPU_HOP_INT || code == MZGPU_HOP_MAP) {
      v[sp] = code == MZGPU_HOP_INT ? consts[o.konst].lo : code == MZGPU_HOP_MAP ? mv[o.arg] : mfp_field(w, o);
      err[sp] = 0;
      pay[sp] = 0;
      ++sp;
      continue;
    }
    const int y = sp - 1;
    if (code == MZGPU_HOP_NOT) {
      if (err[y] == 0) v[y] ^= 1;
      continue;
    }
    if ((code >= MZGPU_HOP_INT_TO_MZTS && code <= MZGPU_HOP_DATE_TO_MZTS) || code == MZGPU_HOP_NEG ||
        code == MZGPU_HOP_ABS || code == MZGPU_HOP_INT64_TO_INT32) {  // the unary ops and TS + interval
      if (err[y] != 0) continue;
      const i64 a = (i64)v[y];
      if (code == MZGPU_HOP_INT_TO_MZTS || code == MZGPU_HOP_TS_TO_MZTS || code == MZGPU_HOP_DATE_TO_MZTS) {
        i64 r = a;
        if (code == MZGPU_HOP_TS_TO_MZTS) r = a >= 0 ? a / 1000 : -((-(a + 1)) / 1000) - 1;  // toward -inf
        if (code == MZGPU_HOP_DATE_TO_MZTS) r = a * 86400000ll;                             // i32 days: no overflow
        if (r < 0) {
          err[y] = MZGPU_MFP_ERR_MZ_TIMESTAMP_OUT_OF_RANGE;
          pay[y] = (u64)a;
        } else {
          v[y] = (u64)r;
        }
      } else if (code == MZGPU_HOP_TS_ADD_IV) {  // the interval is folded to i64 microseconds on the host
        const i64 b = iv_us[o.konst];
        const i64 r = (i64)((u64)a + (u64)b);
        if ((((a ^ r) & (b ^ r)) < 0) || r < TS_LOW_US || r > TS_HIGH_US) {
          err[y] = MZGPU_MFP_ERR_TIMESTAMP_OUT_OF_RANGE;
          pay[y] = 0;
        } else {
          v[y] = (u64)r;
        }
      } else if (code == MZGPU_HOP_INT64_TO_INT32) {
        if (a != (i64)(int)a) {
          err[y] = MZGPU_HAVING_ERR_INT32_OUT_OF_RANGE;
          pay[y] = (u64)a;
        }
      } else {  // NEG / ABS: checked_neg / checked_abs at width arg
        const i64 lo = o.arg == 32 ? (i64)(-2147483647 - 1) : (i64)0x8000000000000000ull;
        if (a == lo) {
          err[y] = o.arg == 32 ? MZGPU_HAVING_ERR_INT32_OUT_OF_RANGE : MZGPU_HAVING_ERR_INT64_OUT_OF_RANGE;
          pay[y] = (u64)a;
        } else if (code == MZGPU_HOP_NEG || a < 0) {
          v[y] = (u64)0 - (u64)a;
        }
      }
      continue;
    }
    if (code == MZGPU_HOP_IF) {  // c, t, e: the condition's error, else the taken branch's value or error
      sp -= 2;
      const int c = sp - 1, t = sp, e = sp + 1;
      if (err[c] == 0) {
        const int k = v[c] == 1 ? t : e;
        v[c] = v[k];
        err[c] = err[k];
        pay[c] = pay[k];
      }
      continue;
    }
    --sp;
    const int x = sp - 1;
    const u32 ex = err[x], ey = err[y];
    if (code == MZGPU_HOP_AND || code == MZGPU_HOP_OR) {
      // variadic And / Or: the dominant value wins over an error, else the larger error (of one code, the
      // payload-0 one: a division's "a / b" message orders after NEG / ABS's operand)
      const u64 dom = code == MZGPU_HOP_AND ? 0 : 1;
      if ((ex == 0 && v[x] == dom) || (ey == 0 && v[y] == dom)) {
        v[x] = dom;
        err[x] = 0;
      } else if (ey > ex || (ey != 0 && ey == ex && pay[y] == 0)) {
        err[x] = ey;
        pay[x] = pay[y];
      }
      continue;
    }
    if (ex != 0 || ey != 0) {  // the first operand's error, else the second's
      if (ex == 0) {
        err[x] = ey;
        pay[x] = pay[y];
      }
      continue;
    }
    if (code == MZGPU_HOP_CMP) {
      const i64 a = (i64)v[x], b = (i64)v[y];
      bool r;
      switch (o.arg) {
        case MZGPU_CMP_EQ: r = a == b; break;
        case MZGPU_CMP_NE: r = a != b; break;
        case MZGPU_CMP_LT: r = a < b; break;
        case MZGPU_CMP_LE: r = a <= b; break;
        case MZGPU_CMP_GT: r = a > b; break;
        default: r = a >= b; break;
      }
      v[x] = r ? 1 : 0;
      continue;
    }
    i64 r = 0;
    const u32 e = mfp_arith(code, o.arg, (i64)v[x], (i64)v[y], &r);
    if (e != 0) {
      err[x] = e;
      pay[x] = 0;
    } else {
      v[x] = (u64)r;
    }
  }
  MVal out;
  out.v = v[0];
  out.err = err[0];
  out.pay = pay[0];
  return out;
}

// inclusive warp scan of small counts; returns the exclusive prefix, *total = the warp's sum
__device__ __forceinline__ u32 warp_excl(u32 c, u32* total) {
  const int lane = threadIdx.x & 31;
  u32 s = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u32 t = __shfl_up_sync(0xffffffffu, s, d);
    if (lane >= d) s += t;
  }
  *total = __shfl_sync(0xffffffffu, s, 31);
  return s - c;
}

// one warp-aggregated reservation of `c` rows at *cursor
__device__ __forceinline__ u64 warp_reserve(u32 c, unsigned long long* cursor) {
  u32 total;
  const u32 ex = warp_excl(c, &total);
  u64 base = 0;
  if ((threadIdx.x & 31) == 31 && total) base = atomicAdd(cursor, (unsigned long long)total);
  base = __shfl_sync(0xffffffffu, base, 31);
  return base + ex;
}

// The non-temporal half of MfpPlan::evaluate over the words w (SafeMfpPlan::evaluate_inner): each predicate after
// the expressions below its support, in order, then every remaining expression; mv receives the expression values.
// Returns whether the row survives; an error stops evaluation and is left in *e_code / *e_pay.
__device__ __forceinline__ bool mfp_filter_map(const MfpDevPlan& pl, const u64* w, u64* mv, u32* e_code,
                                               u64* e_pay) {
  bool keep = true;
  u32 ne = 0;
  // the expressions below `support`, in index order; an error stops the row
  auto eval_maps = [&](u32 support) {
    for (; ne < support && keep; ++ne) {
      const MVal m = mfp_run(pl.map.ops[ne], pl.map.n_ops[ne], pl.map.consts, pl.map_iv_us, w, mv);
      if (m.err) {
        *e_code = m.err;
        *e_pay = m.pay;
        keep = false;
      }
      mv[ne] = m.v;
    }
  };
  for (u32 p = 0; p < pl.plan.n_predicates && keep; ++p) {
    eval_maps(pl.support[p]);
    if (!keep) break;
    const MVal m = mfp_run(pl.plan.ops[p], pl.plan.n_ops[p], pl.plan.consts, pl.iv_us, w, mv);
    if (m.err) {
      *e_code = m.err;
      *e_pay = m.pay;
      keep = false;
    } else if (m.v == 0) {
      keep = false;
    }
  }
  eval_maps(pl.map.n_exprs);
  return keep;
}

// The projection: the first ONW - 2 output words over the words w and the expression values mv.
template <int ONW>
__device__ __forceinline__ void mfp_project(const MfpDevPlan& pl, const u64* w, const u64* mv, u64* o) {
#pragma unroll
  for (int k = 0; k < ONW - 2; ++k) {
    u64 acc = 0;
    for (u32 f = 0; f < pl.plan.n_fields[k]; ++f) {
      const mzgpu_field fd = pl.plan.fields[k][f];
      u64 a = (fd.src >= MZGPU_SRC_MAP0 ? mv[fd.src - MZGPU_SRC_MAP0] : w[fd.src]) >> fd.shift;
      if (fd.bits < 64) a &= (1ull << fd.bits) - 1;
      acc |= a << fd.dst_shift;
    }
    o[k] = acc;
  }
}

}  // namespace
#endif  // __CUDACC__
