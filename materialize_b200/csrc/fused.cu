// fused.cu — "consolidate" as ONE cooperative kernel with every size read on the
// device: sort + diff-sum + zero-drop, optionally over the union of two sorted
// inputs with times advanced (batch merge), optionally split by a frontier
// (batcher seal), optionally followed by the hash index of the result.
//
// Reference semantics (same as sort.cu / consolidate.cu / merge.cu / index.cu):
//   consolidate_updates               differential-dataflow 0.23 (ext), model at
//                                     src/timely-util/src/columnar/batcher.rs:1116-1130
//   Chunker::push_into + seal/extract src/timely-util/src/columnar/batcher.rs:65-122,
//                                     src/timely-util/src/columnation.rs:636-655
//   Batch::Merger (advance_by(since)) SURVEY.md A4
//
// Why one kernel: a 100K-row update batch (BASELINE config 3) moves ~3 MB; each
// of the ~25 kernels of the unfused path runs for microseconds and three of them
// end in a host read-back.  Here a persistent grid runs every phase back to back
// with a device-side grid barrier between phases; the input row count is read
// from device memory (DLen) and every result count (rows out, keys, longest key
// run, rows kept, min kept time) is left in a device counter block (Lazy4), so
// the host enqueues the launch and moves on.  CTAs beyond what the actual row
// count needs leave at once, so a loose upper bound costs nothing.
//
//   phase 0  zero scratch, min/max of every key word (times advanced by `since`)
//   plan     (every CTA, identical) radix rounds of <= 64 composite bits, least
//            significant key words first
//   round r  pack composites (+ all-digit histogram) | scan | 8-bit passes with
//            decoupled look-back (radix.cuh)
//   gather   rows by the final permutation, head flags
//   segsum   warp-segmented diff sums, one atomic per (warp, segment)
//   count    surviving segments per tile, split into ship (time < upper) / keep
//   emit     ship rows -> out, kept rows -> keep
//   index    open-addressing hash index over the distinct keys of `out`
#include "common.cuh"
#include "radix.cuh"

namespace {

constexpr int FT = RS_THREADS;  // 256 threads per CTA
constexpr int FI = 4;           // radix items per thread: 1024-key tiles
constexpr int FTILE = FT * FI;
constexpr int MAX_ROUNDS = 6;
constexpr u32 MAX_RUN_SAT = 1024;  // key runs longer than this report as 1024
// MSD path: rows are partitioned into buckets by the leading bits of their
// composite key and every bucket is sorted AND consolidated inside one CTA's
// shared memory (rows with equal keys always share a bucket).
constexpr u32 MSD_MAX_BUCKETS = 4096;        // exact (count -> scan -> scatter) MSD path: bucket bases live in shared memory
constexpr u32 MSD_FAST_MAX_BUCKETS = 32768;  // fast MSD path (fixed-capacity regions): up to 2^20 rows at 32-48 rows per bucket
constexpr u64 MSD_FAST_MAX_ROWS = 1ull << 20;
constexpr u64 MSD_EXACT_MAX_ROWS = 1ull << 18;
constexpr u32 MSD_LOCAL_MAX = 1024;  // largest bucket the in-CTA sort takes

struct FusedCtl {
  u32 barrier;
  u32 overflow;  // fast MSD path: a bucket outgrew its fixed-capacity region (the exact path runs instead)
  u32 pad[2];
  u64 minmax[12];  // [2k] = max of ~word (so zero is the identity), [2k+1] = max of word
  u64 n_seg;
  u64 n_out;
  u32 hist[MAX_ROUNDS * 8 * 256];
  u32 bcnt[MSD_FAST_MAX_BUCKETS];  // MSD paths: rows per bucket
};
constexpr size_t CTL_HEADER = offsetof(FusedCtl, hist);

struct FusedArgs {
  const u64* a;
  const u64* b;
  DLen na, nb;
  u64 since, upper;
  FusedCtl* ctl;
  FusedCtl* ctl_next;  // header zeroed here for the next launch
  u64* k0;
  u64* k1;
  u32* v0;
  u32* v1;
  u32* state0;  // [Tcap][256]
  u32* state1;
  u64* sorted;     // cap rows
  u32* tile_cnt;   // [Ucap]
  u32* tile_cnt2;  // [Ucap]
  u64* seg_sums;   // [cap][ND]
  u32* seg_first;  // [cap]
  u64* out;        // cap rows
  u64* keep;       // cap rows or null
  HashSlot* table;  // table_cap slots or null
  u64 table_cap;
  u64* res;   // n_out, mask, n_keys, max_run
  u64* kres;  // n_keep, min kept time, max input time, -
  u64* dbg;   // optional: CTA 0 leaves a globaltimer stamp per phase (profiling runs only)
  u64* m_lo;  // MSD path: composites and row indices grouped by bucket (cap each)
  u64* m_hi;
  u32* m_idx;
  u64* lb_ship;  // MSD path: look-back state per bucket ((ship << 21) | keep counts), zeroed in phase 0
  u64* lb_keep;
  u32 max_g;     // CTAs that take part at most
  u32 merge;     // both inputs are sorted and consolidated: merge path instead of a sort
  u32 fast;      // fast MSD path allowed (fused_prepare always sets it)
  u32 merge_sort_max;  // a merge of at most this many rows runs as a sort of A ++ B (MERGE_SORT_MAX)
};

__device__ __forceinline__ u64 gtimer() {
  u64 t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define PHASE_STAMP(i)                                                \
  do {                                                                \
    if (a.dbg != nullptr && c == 0 && tid == 0) a.dbg[(i)] = gtimer(); \
  } while (0)

// Grid-wide barrier over the job's own counter (monotone: epoch e completes at e * G arrivals).
// One thread per CTA arrives with a release reduction and spins on an acquire load; the
// __syncthreads() on either side extend the ordering to the whole CTA (CTA-scope barriers are
// cumulative), so everything written before the barrier by any CTA is visible after it.
__device__ __forceinline__ void grid_barrier(u32* counter, u32 G, u32& epoch) {
  __syncthreads();
  epoch++;
  if (threadIdx.x == 0) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
    const u32 target = epoch * G;
    u32 v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    } while (v < target);
  }
  __syncthreads();
}

__device__ __forceinline__ int bit_width_dev(u64 x) { return x == 0 ? 0 : 64 - __clzll((long long)x); }

// sum of a u32 array prefix [0, m) by the whole CTA
__device__ __forceinline__ u32 block_sum_prefix(const u32* a, u64 m, u32* sm) {
  u32 v = 0;
  for (u64 i = threadIdx.x; i < m; i += FT) v += *(volatile const u32*)(a + i);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  if (lane_id() == 0) sm[warp_id()] = v;
  __syncthreads();
  u32 tot = 0;
  for (int w = 0; w < FT / 32; ++w) tot += sm[w];
  __syncthreads();
  return tot;
}

struct MsdSmem {
  u64 lo[MSD_LOCAL_MAX];
  u64 hi[MSD_LOCAL_MAX];
  u32 idx[MSD_LOCAL_MAX];
  u64 sum[MSD_LOCAL_MAX];  // one-word diff sums per segment of the bucket
  u64 sum8[256][8];        // accumulable diffs (8 words): buckets of at most 256 rows
};
struct MsdScan {  // phase "scatter": bucket bases
  u32 base[MSD_MAX_BUCKETS + 1];
};

// logical input row i of A ++ B, time advanced to max(time, since)
template <int RB>
__device__ __forceinline__ void load_in_row(const FusedArgs& a, u64 na, u64 since, u64 i, u64* r) {
  constexpr int NW = RowT<RB>::NW, TW = RowT<RB>::TW;
  if (i < na)
    load_row<NW>(a.a, i, r);
  else
    load_row<NW>(a.b, i - na, r);
  if (TW >= 0) {
    u64& t = r[TW >= 0 ? TW : 0];
    t = t < since ? since : t;
  }
}

// ---- MSD bucket phase, one bucket per WARP (buckets of at most 32*R rows): the
// bucket's composites live in registers, a shuffle bitonic network sorts them,
// a warp-segmented scan sums the diffs of equal keys, and the surviving rows are
// emitted at offsets from a look-back over chunks of eight buckets (one chunk per
// CTA iteration).  No shared-memory sort, no block-wide scans: ~5 us per chunk.
template <int RB, int R>
__device__ __forceinline__ void msd_warp_buckets(const FusedArgs& a, FusedCtl* ctl, const u32* base, u32 NB, u32 c,
                                                 u32 G, u64 na, u64 since, u64* s_cnt /* 8 + 1 words */,
                                                 u64* s_lb) {
  constexpr int NW = RowT<RB>::NW, NK = RowT<RB>::NK, ND = RowT<RB>::ND, TW = RowT<RB>::TW;
  const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const u64 upper = a.upper;
  LookBack lbs;
  lbs.state = a.lb_ship;
  lbs.ticket = nullptr;
  lbs.epoch = 1;
  const u32 n_chunks = (NB + 7) / 8;
  for (u32 ch = c; ch < n_chunks; ch += G) {
    const u32 b = ch * 8 + warp;
    u32 gbase = 0, m = 0;
    if (b < NB) {
      gbase = base[b];
      m = base[b + 1] - gbase;
    }
    u64 hi[R], lo[R];
    u32 ix[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const u32 p = r * 32 + lane;
      if (p < m) {
        lo[r] = a.m_lo[gbase + p];
        hi[r] = a.m_hi[gbase + p];
        ix[r] = a.m_idx[gbase + p];
      } else {
        lo[r] = ~0ull;
        hi[r] = ~0ull;
        ix[r] = 0xffffffffu;
      }
    }
    // diffs (and time) of the rows as they arrived; they travel with the sort
    // bitonic network over positions p = r*32 + lane, ordered by (hi, lo, idx)
#pragma unroll
    for (int k = 2; k <= 32 * R; k <<= 1) {
#pragma unroll
      for (int j = k >> 1; j > 0; j >>= 1) {
        if (j >= 32) {
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const int r2 = r ^ (j >> 5);
            if (r2 > r) {
              const bool up = (((r * 32 + (int)lane) & k) == 0);
              const bool gt = hi[r] > hi[r2] || (hi[r] == hi[r2] && (lo[r] > lo[r2] || (lo[r] == lo[r2] && ix[r] > ix[r2])));
              if (gt == up) {
                u64 t0 = hi[r];
                hi[r] = hi[r2];
                hi[r2] = t0;
                t0 = lo[r];
                lo[r] = lo[r2];
                lo[r2] = t0;
                u32 t1 = ix[r];
                ix[r] = ix[r2];
                ix[r2] = t1;
              }
            }
          }
        } else {
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const u64 ohi = __shfl_xor_sync(0xffffffffu, hi[r], j);
            const u64 olo = __shfl_xor_sync(0xffffffffu, lo[r], j);
            const u32 oix = __shfl_xor_sync(0xffffffffu, ix[r], j);
            const bool up = (((r * 32 + (int)lane) & k) == 0);
            const bool lower = ((lane & j) == 0);
            const bool gt = hi[r] > ohi || (hi[r] == ohi && (lo[r] > olo || (lo[r] == olo && ix[r] > oix)));
            // the lower position keeps the smaller element when ascending
            const bool take = (lower == up) ? gt : !gt;
            if (take) {
              hi[r] = ohi;
              lo[r] = olo;
              ix[r] = oix;
            }
          }
        }
      }
    }
    // head flags, diffs
    bool head[R];
    u64 d[R][ND];
    u64 tt[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const u32 p = r * 32 + lane;
      u64 phi = __shfl_up_sync(0xffffffffu, hi[r], 1), plo = __shfl_up_sync(0xffffffffu, lo[r], 1);
      if (r > 0) {
        const u64 qhi = __shfl_sync(0xffffffffu, hi[r - 1 >= 0 ? r - 1 : 0], 31);
        const u64 qlo = __shfl_sync(0xffffffffu, lo[r - 1 >= 0 ? r - 1 : 0], 31);
        if (lane == 0) {
          phi = qhi;
          plo = qlo;
        }
      }
      head[r] = p < m && (p == 0 || phi != hi[r] || plo != lo[r]);
      tt[r] = 0;
      if (p < m) {
        u64 row[NW];
        load_in_row<RB>(a, na, since, ix[r], row);
#pragma unroll
        for (int w = 0; w < ND; ++w) d[r][w] = row[NK + w];
        if (TW >= 0) tt[r] = row[TW >= 0 ? TW : 0];
      } else {
#pragma unroll
        for (int w = 0; w < ND; ++w) d[r][w] = 0;
      }
    }
    // segmented inclusive sums in position order; the carry crosses register rows
    u64 carry[ND];
#pragma unroll
    for (int w = 0; w < ND; ++w) carry[w] = 0;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const u32 hm = __ballot_sync(0xffffffffu, head[r]);
      const u32 below = hm & (lane == 31 ? 0xffffffffu : ((2u << lane) - 1));
      const int my_start = below ? 31 - __clz(below) : -1;  // lane of my segment's head in this row (-1: continues)
      const int start_eff = my_start < 0 ? 0 : my_start;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        u64 o[ND];
#pragma unroll
        for (int w = 0; w < ND; ++w) o[w] = __shfl_up_sync(0xffffffffu, d[r][w], off);
        if ((int)lane - off >= start_eff) diff_add<ND>(d[r], o);
      }
      if (my_start < 0) diff_add<ND>(d[r], carry);  // my segment started in an earlier row
#pragma unroll
      for (int w = 0; w < ND; ++w) carry[w] = __shfl_sync(0xffffffffu, d[r][w], 31);
    }
    // survivors: the LAST row of every segment carries the segment's sum
    u32 cls[R];
    u32 cnt_ship = 0, cnt_keep = 0;
    u32 pos_ship[R], pos_keep[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const u32 p = r * 32 + lane;
      bool nhead = __shfl_down_sync(0xffffffffu, head[r], 1);
      if (r + 1 < R) {
        const bool q = __shfl_sync(0xffffffffu, head[r + 1 < R ? r + 1 : r], 0);
        if (lane == 31) nhead = q;
      } else if (lane == 31) {
        nhead = true;
      }
      const bool tail = p < m && (p == m - 1 || nhead);
      cls[r] = 0;
      if (tail && !diff_is_zero<ND>(d[r]))
        cls[r] = (TW < 0 || upper == MZGPU_FRONTIER_EMPTY || tt[r] < upper) ? 1u : 2u;
      const u32 ms = __ballot_sync(0xffffffffu, cls[r] == 1u), mk = __ballot_sync(0xffffffffu, cls[r] == 2u);
      const u32 lt = (1u << lane) - 1;
      pos_ship[r] = cnt_ship + __popc(ms & lt);
      pos_keep[r] = cnt_keep + __popc(mk & lt);
      cnt_ship += __popc(ms);
      cnt_keep += __popc(mk);
    }
    // chunk-level offsets: eight warps, then the look-back over chunks
    __syncthreads();
    if (lane == 0) s_cnt[warp] = ((u64)cnt_ship << 21) | (u64)cnt_keep;
    __syncthreads();
    u64 mine = 0, total = 0;
#pragma unroll
    for (int w = 0; w < FT / 32; ++w) {
      const u64 v = s_cnt[w];
      if ((u32)w < warp) mine += v;
      total += v;
    }
    const u64 chunk_base = lb_exclusive_prefix(lbs, ch, total, s_lb);
    const u64 bases = chunk_base + mine;
    const u64 ship_base = bases >> 21, keep_base = bases & ((1ull << 21) - 1);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (cls[r] != 0u) {
        u64 row[NW];
        load_in_row<RB>(a, na, since, ix[r], row);
#pragma unroll
        for (int w = 0; w < ND; ++w) row[NK + w] = d[r][w];
        if (cls[r] == 1u) {
          store_row<NW>(a.out, ship_base + pos_ship[r], row);
        } else if (a.keep != nullptr) {
          store_row<NW>(a.keep, keep_base + pos_keep[r], row);
          if (TW >= 0) atomicMin((unsigned long long*)&a.kres[1], (unsigned long long)row[TW >= 0 ? TW : 0]);
        }
      }
    }
    if (ch == n_chunks - 1 && tid == 0) {
      const u64 all = chunk_base + total;
      ctl->n_out = all >> 21;
      a.res[0] = all >> 21;
      a.kres[0] = all & ((1ull << 21) - 1);
    }
  }
}

// ---- fast MSD path, bucket phase.  Differences from msd_warp_buckets above:
//  * a bucket is a FIXED-capacity region (32*R slots at b * 32*R) that the pack phase filled
//    directly (slot = atomic counter of the bucket), so there is no count -> scan -> scatter;
//  * only the bits that vary inside a bucket are kept (the composite minus its leading bucket
//    bits): KW = 1 when they fit one word -- the usual case -- halves the sort's shuffles;
//  * the hash index of the shipped rows is built right here when a key cannot span buckets
//    (`inline_index`): the warp knows the final position of every row it ships once the
//    look-back has given the chunk's base, so no table pass (and no grid barrier) follows.
template <int RB, int R, int KW>
__device__ __forceinline__ void msd_warp_buckets2(const FusedArgs& a, FusedCtl* ctl, u32 NB, u32 c, u32 G, u64 na,
                                                  u64 since, u64 mask, bool inline_index, u64* s_cnt, u64* s_lb,
                                                  u64* s_keys /* [FT/32][32*R] */, u32* s_stat /* [2] */) {
  constexpr int NW = RowT<RB>::NW, NK = RowT<RB>::NK, ND = RowT<RB>::ND, TW = RowT<RB>::TW;
  constexpr u32 CAP = 32u * R;
  const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const u64 upper = a.upper;
  LookBack lbs;
  lbs.state = a.lb_ship;
  lbs.ticket = nullptr;
  lbs.epoch = 1;
  u64* wkeys = s_keys + (size_t)warp * CAP;
  u32 my_heads = 0, my_run = 0;
  const u32 n_chunks = (NB + 7) / 8;
  for (u32 ch = c; ch < n_chunks; ch += G) {
    const u32 b = ch * 8 + warp;
    u32 m = 0;
    if (b < NB) {
      m = *(volatile u32*)&ctl->bcnt[b];
      m = m < CAP ? m : CAP;  // (an overflow never gets here: the exact path runs instead)
    }
    const u64 gbase = (u64)b * CAP;
    u64 hi[R], lo[R];
    u32 ix[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const u32 p = r * 32 + lane;
      if (p < m) {
        lo[r] = a.m_lo[gbase + p];
        hi[r] = KW == 2 ? a.m_hi[gbase + p] : 0ull;
        ix[r] = a.m_idx[gbase + p];
      } else {
        lo[r] = ~0ull;
        hi[r] = KW == 2 ? ~0ull : 0ull;
        ix[r] = 0xffffffffu;
      }
    }
    // bitonic network over positions p = r*32 + lane, ordered by (hi, lo, idx): idx makes real
    // elements distinct (and puts the padding last among equal keys).  The (k, j) stages are
    // LOOPS: fully unrolled the network is ~2K instructions that every warp runs through once,
    // and the kernel stalls on instruction fetch.
    // Stages with j >= 32 exchange whole register rows (static pairs), the others shuffle.
    auto greater = [&](u64 h1, u64 l1, u32 i1, u64 h2, u64 l2, u32 i2) -> bool {
      if (KW == 2) return h1 > h2 || (h1 == h2 && (l1 > l2 || (l1 == l2 && i1 > i2)));
      return l1 > l2 || (l1 == l2 && i1 > i2);
    };
    auto local_exchange = [&](int r, int r2, int k) {
      const bool up = (((r * 32 + (int)lane) & k) == 0);
      if (greater(hi[r], lo[r], ix[r], hi[r2], lo[r2], ix[r2]) == up) {
        u64 t0 = lo[r];
        lo[r] = lo[r2];
        lo[r2] = t0;
        if (KW == 2) {
          t0 = hi[r];
          hi[r] = hi[r2];
          hi[r2] = t0;
        }
        const u32 t1 = ix[r];
        ix[r] = ix[r2];
        ix[r2] = t1;
      }
    };
#pragma unroll 1
    for (int k = 2; k <= 32 * R; k <<= 1) {
#pragma unroll 1
      for (int j = k >> 1; j > 0; j >>= 1) {
        if (j >= 32) {
          // R <= 4: j == 64 pairs rows (0,2),(1,3); j == 32 pairs (0,1),(2,3)
          if (j == 64) {
            if (R >= 4) {
              local_exchange(0, 2 < R ? 2 : 0, k);
              local_exchange(1 < R ? 1 : 0, 3 < R ? 3 : 0, k);
            }
          } else {
            if (R >= 2) local_exchange(0, 1 < R ? 1 : 0, k);
            if (R >= 4) local_exchange(2 < R ? 2 : 0, 3 < R ? 3 : 0, k);
          }
        } else {
          const bool lower = ((lane & j) == 0);
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const u64 olo = __shfl_xor_sync(0xffffffffu, lo[r], j);
            const u64 ohi = KW == 2 ? __shfl_xor_sync(0xffffffffu, hi[r], j) : 0ull;
            const u32 oix = __shfl_xor_sync(0xffffffffu, ix[r], j);
            const bool up = (((r * 32 + (int)lane) & k) == 0);
            const bool gt = greater(hi[r], lo[r], ix[r], ohi, olo, oix);
            const bool take = (lower == up) ? gt : !gt;
            if (take) {
              lo[r] = olo;
              if (KW == 2) hi[r] = ohi;
              ix[r] = oix;
            }
          }
        }
      }
    }
    // head flags, diffs
    bool head[R];
    u64 d[R][ND];
    u64 tt[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const u32 p = r * 32 + lane;
      u64 plo = __shfl_up_sync(0xffffffffu, lo[r], 1);
      u64 phi = KW == 2 ? __shfl_up_sync(0xffffffffu, hi[r], 1) : 0ull;
      if (r > 0) {
        const u64 qlo = __shfl_sync(0xffffffffu, lo[r - 1 >= 0 ? r - 1 : 0], 31);
        const u64 qhi = KW == 2 ? __shfl_sync(0xffffffffu, hi[r - 1 >= 0 ? r - 1 : 0], 31) : 0ull;
        if (lane == 0) {
          plo = qlo;
          phi = qhi;
        }
      }
      head[r] = p < m && (p == 0 || plo != lo[r] || (KW == 2 && phi != hi[r]));
      tt[r] = 0;
      if (p < m) {
        u64 row[NW];
        load_in_row<RB>(a, na, since, ix[r], row);
#pragma unroll
        for (int w = 0; w < ND; ++w) d[r][w] = row[NK + w];
        if (TW >= 0) tt[r] = row[TW >= 0 ? TW : 0];
      } else {
#pragma unroll
        for (int w = 0; w < ND; ++w) d[r][w] = 0;
      }
    }
    // segmented inclusive sums in position order; the carry crosses register rows
    u64 carry[ND];
#pragma unroll
    for (int w = 0; w < ND; ++w) carry[w] = 0;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const u32 hm = __ballot_sync(0xffffffffu, head[r]);
      const u32 below = hm & (lane == 31 ? 0xffffffffu : ((2u << lane) - 1));
      const int my_start = below ? 31 - __clz(below) : -1;
      const int start_eff = my_start < 0 ? 0 : my_start;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        u64 o[ND];
#pragma unroll
        for (int w = 0; w < ND; ++w) o[w] = __shfl_up_sync(0xffffffffu, d[r][w], off);
        if ((int)lane - off >= start_eff) diff_add<ND>(d[r], o);
      }
      if (my_start < 0) diff_add<ND>(d[r], carry);
#pragma unroll
      for (int w = 0; w < ND; ++w) carry[w] = __shfl_sync(0xffffffffu, d[r][w], 31);
    }
    // survivors: the LAST row of every segment carries the segment's sum
    u32 cls[R];
    u32 cnt_ship = 0, cnt_keep = 0;
    u32 pos_ship[R], pos_keep[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const u32 p = r * 32 + lane;
      bool nhead = __shfl_down_sync(0xffffffffu, head[r], 1);
      if (r + 1 < R) {
        const bool q = __shfl_sync(0xffffffffu, head[r + 1 < R ? r + 1 : r], 0);
        if (lane == 31) nhead = q;
      } else if (lane == 31) {
        nhead = true;
      }
      const bool tail = p < m && (p == m - 1 || nhead);
      cls[r] = 0;
      if (tail && !diff_is_zero<ND>(d[r]))
        cls[r] = (TW < 0 || upper == MZGPU_FRONTIER_EMPTY || tt[r] < upper) ? 1u : 2u;
      const u32 ms = __ballot_sync(0xffffffffu, cls[r] == 1u), mk = __ballot_sync(0xffffffffu, cls[r] == 2u);
      const u32 lt = (1u << lane) - 1;
      pos_ship[r] = cnt_ship + __popc(ms & lt);
      pos_keep[r] = cnt_keep + __popc(mk & lt);
      cnt_ship += __popc(ms);
      cnt_keep += __popc(mk);
    }
    // chunk-level offsets: eight warps, then the look-back over chunks
    __syncthreads();
    if (lane == 0) s_cnt[warp] = ((u64)cnt_ship << 21) | (u64)cnt_keep;
    __syncthreads();
    u64 mine = 0, total = 0;
#pragma unroll
    for (int w = 0; w < FT / 32; ++w) {
      const u64 v = s_cnt[w];
      if ((u32)w < warp) mine += v;
      total += v;
    }
    const u64 chunk_base = lb_exclusive_prefix(lbs, ch, total, s_lb);
    const u64 bases = chunk_base + mine;
    const u64 ship_base = bases >> 21, keep_base = bases & ((1ull << 21) - 1);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (cls[r] != 0u) {
        u64 row[NW];
        load_in_row<RB>(a, na, since, ix[r], row);
#pragma unroll
        for (int w = 0; w < ND; ++w) row[NK + w] = d[r][w];
        if (cls[r] == 1u) {
          store_row<NW>(a.out, ship_base + pos_ship[r], row);
          if (inline_index) wkeys[pos_ship[r]] = row[0];
        } else if (a.keep != nullptr) {
          store_row<NW>(a.keep, keep_base + pos_keep[r], row);
          if (TW >= 0) atomicMin((unsigned long long*)&a.kres[1], (unsigned long long)row[TW >= 0 ? TW : 0]);
        }
      }
    }
    if (inline_index) {
      // keys of the rows this warp shipped, in output order: heads claim their slots
      __syncwarp();
      for (u32 e = lane; e < cnt_ship; e += 32) {
        const u64 key = wkeys[e];
        if (e == 0 || wkeys[e - 1] != key) {
          u32 run = 1;
          while (e + run < cnt_ship && wkeys[e + run] == key) ++run;
          ++my_heads;
          my_run = run > my_run ? run : my_run;
          const u64 meta = (ship_base + e + 1) | ((u64)(run < MAX_RUN_SAT ? run : 0u) << 44);
          u64 h = mix64(key) & mask;
          while (true) {
            unsigned long long prev = atomicCAS((unsigned long long*)&a.table[h].meta, 0ull, (unsigned long long)meta);
            if (prev == 0ull) {
              a.table[h].key = key;
              break;
            }
            h = (h + 1) & mask;
          }
        }
      }
      __syncwarp();
    }
    if (ch == n_chunks - 1 && tid == 0) {
      const u64 all = chunk_base + total;
      ctl->n_out = all >> 21;
      a.res[0] = all >> 21;
      a.kres[0] = all & ((1ull << 21) - 1);
    }
  }
  if (inline_index) {
    // distinct keys and the longest key run: one global atomic each per CTA
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      my_heads += __shfl_xor_sync(0xffffffffu, my_heads, off);
      const u32 o = __shfl_xor_sync(0xffffffffu, my_run, off);
      my_run = o > my_run ? o : my_run;
    }
    if (lane == 0) {
      if (my_heads) atomicAdd(&s_stat[0], my_heads);
      if (my_run) atomicMax(&s_stat[1], my_run);
    }
    __syncthreads();
    if (tid == 0) {
      if (s_stat[0]) atomicAdd((unsigned long long*)&a.res[2], (unsigned long long)s_stat[0]);
      if (s_stat[1]) atomicMax((unsigned long long*)&a.res[3], (unsigned long long)s_stat[1]);
    }
  }
}

union FusedSmem {
  RsSmemT<FI> rs;
  u32 hist[8 * 256];
  MsdSmem msd;
  MsdScan scan;
  u64 wkeys[FT / 32][128];  // fast MSD path: keys of the rows a warp ships (inline hash index)
};

// The whole operator for one job.  `c` = this CTA's index among the `gdim` CTAs the launch gave
// the job (a single-job launch: blockIdx.x / gridDim.x; a multi-job launch: the job's slice of
// the grid).  Every grid-wide step synchronises on the job's own control block, so independent
// jobs of one launch never wait for each other.
template <int RB>
__device__ __forceinline__ void fused_body(const FusedArgs& a, const u32 c, const u32 gdim) {
  constexpr int NW = RowT<RB>::NW, NK = RowT<RB>::NK, ND = RowT<RB>::ND, TW = RowT<RB>::TW;
  __shared__ FusedSmem sm;
  __shared__ u32 sm_scan[34];
  __shared__ int s_nwords, s_nrounds, s_word[6], s_shift[6], s_round[6], s_rbits[MAX_ROUNDS];
  __shared__ int s_shift128[6], s_w128, s_keybits;
  __shared__ u32 s_max_bucket, s_max_unit;
  __shared__ u64 s_minv[6];
  const u32 tid = threadIdx.x;
  const u64 na = dlen_get(a.na), nb = dlen_get(a.nb);
  const u64 n = na + nb;
  const u64 T = (n + FTILE - 1) / FTILE;
  // A merge of update-batch size runs as a sort of A ++ B: the fast MSD path below has two grid
  // barriers, the merge path five; sortedness only pays beyond the bucket phase's reach.
  const bool merge = a.merge != 0 && !(a.fast != 0 && n <= (u64)a.merge_sort_max);
  // CTAs the actual input needs; the rest leave (they hold no barrier slot)
  // MSD bucket count from the row count alone: at most 48 (12 for the 80-byte
  // accumulable rows, whose warp capacity is 64 and whose keys arrive in clumps:
  // one row per lineitem of an order) rows per bucket on average
  constexpr int WR = 4;                     // register rows per lane in the warp-bucket phase
  constexpr u32 WCAP = 32u * WR;            // largest bucket a warp takes
  u32 bb = 0;  // log2(buckets)
  // (the fast path takes up to 32768 buckets -- a million rows; without it the exact path's 4096)
  const u32 bb_max = a.fast != 0 ? 15u : 12u;
  while (bb < bb_max && ((u64)(ND >= 8 ? 12 : 48) << bb) < n) ++bb;
  const u32 NB = 1u << bb;
  u32 G = gdim;
  {
    // the bucket phase of the MSD path wants one CTA per bucket; a merge only has its
    // 1024-row tiles (fewer CTAs = cheaper grid barriers)
    // (a merge has no buckets: two 256-row tiles of the consolidation tail per CTA)
    const u64 half_u = (n + 2 * FT - 1) / (2 * FT);
    u64 want = merge ? (half_u > T ? half_u : T) : (T < (u64)((NB + 7) / 8) ? (u64)((NB + 7) / 8) : T);
    if (want == 0) want = 1;
    if (want < (u64)G) G = (u32)want;
    if (G > a.max_g) G = a.max_g;  // more CTAs only make the grid barriers slower
  }
  if (c >= G) return;
  const u64 gtid = (u64)c * FT + tid, gstride = (u64)G * FT;
  FusedCtl* ctl = a.ctl;
  u32 epoch = 0;
  const u64 since = a.since;

  // logical input row i of A ++ B, time advanced to max(time, since)
  auto load_in = [&](u64 i, u64* r) {
    if (i < na)
      load_row<NW>(a.a, i, r);
    else
      load_row<NW>(a.b, i - na, r);
    if (TW >= 0) {
      u64& t = r[TW >= 0 ? TW : 0];
      t = t < since ? since : t;
    }
  };

  // table size from the actual input count
  u64 mask = 0;
  if (a.table != nullptr) {
    u64 slots = 2;
    while (slots < 2 * n) slots <<= 1;
    if (slots > a.table_cap) slots = a.table_cap;  // cannot happen: cap >= n
    mask = slots - 1;
  }

  __shared__ u64 s_mm[FT / 32][2 * NK];
  PHASE_STAMP(0);
  // ---- phase 0: zero scratch, results, next launch's header; min/max of every key word
  {
    if (c == 0) {
      for (u32 i = tid; i < CTL_HEADER / 4; i += FT) ((u32*)a.ctl_next)[i] = 0;
      if (tid == 0) {
        a.res[0] = 0;
        a.res[1] = mask;
        a.res[2] = 0;
        a.res[3] = 0;
        a.kres[0] = 0;
        a.kres[1] = ~0ull;
        a.kres[2] = 0;
        a.kres[3] = 0;
      }
    }
    for (u64 i = gtid; i < (u64)MAX_ROUNDS * 8 * 256; i += gstride) ctl->hist[i] = 0;
    for (u64 i = gtid; i < (u64)NB; i += gstride) ctl->bcnt[i] = 0;
    for (u64 i = gtid; i < (u64)(NB + 7) / 8; i += gstride) {  // look-back state: one word per chunk of eight buckets
      a.lb_ship[i] = 0;
      a.lb_keep[i] = 0;
    }
    for (u64 i = gtid; i < T * 256; i += gstride) a.state0[i] = 0;
    u64 mn[NK], mx[NK];
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      mn[k] = 0;
      mx[k] = 0;
    }
    for (u64 i = gtid; i < (merge ? 0 : n); i += gstride) {
      u64 r[NW];
      load_in(i, r);
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        u64 v = r[k];
        mn[k] = ~v > mn[k] ? ~v : mn[k];
        mx[k] = v > mx[k] ? v : mx[k];
      }
    }
#pragma unroll
    for (int k = 0; k < NK; ++k) {
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        u64 x = __shfl_xor_sync(0xffffffffu, mn[k], off);
        u64 y = __shfl_xor_sync(0xffffffffu, mx[k], off);
        mn[k] = x > mn[k] ? x : mn[k];
        mx[k] = y > mx[k] ? y : mx[k];
      }
      if (lane_id() == 0) {
        s_mm[warp_id()][2 * k] = mn[k];
        s_mm[warp_id()][2 * k + 1] = mx[k];
      }
    }
    // one atomic per CTA and word: same-address atomics from every warp serialise in L2
    __syncthreads();
    if (tid < 2 * NK && n > 0 && !merge) {
      u64 v = 0;
#pragma unroll
      for (int w = 0; w < FT / 32; ++w) v = s_mm[w][tid] > v ? s_mm[w][tid] : v;
      atomicMax((unsigned long long*)&ctl->minmax[tid], (unsigned long long)v);
    }
  }
  // (a merge needs nothing of phase 0 before its own first barrier)
  if (!merge) grid_barrier(&ctl->barrier, G, epoch);

  // ---- plan (every CTA computes the same plan from the global min/max)
  if (tid == 0) {
    int used = 0, nwords = 0, round = 0;
    for (int r = 0; r < MAX_ROUNDS; ++r) s_rbits[r] = 0;
    for (int k = NK - 1; k >= 0; --k) {
      u64 lo = ~*(volatile u64*)&ctl->minmax[2 * k], hi = *(volatile u64*)&ctl->minmax[2 * k + 1];
      int bits = n > 0 ? bit_width_dev(hi - lo) : 0;
      if (bits == 0) continue;
      if (used + bits > 64) {
        round++;
        used = 0;
      }
      s_word[nwords] = k;
      s_shift[nwords] = used;
      s_minv[nwords] = lo;
      s_round[nwords] = round;
      nwords++;
      used += bits;
      s_rbits[round] = used;
    }
    s_nwords = nwords;
    s_nrounds = nwords == 0 ? 0 : round + 1;
    // 128-bit composite layout for the MSD path (least significant word at bit 0)
    int w128 = 0;
    for (int j = 0; j < nwords; ++j) {
      u64 lo = ~*(volatile u64*)&ctl->minmax[2 * s_word[j]], hi = *(volatile u64*)&ctl->minmax[2 * s_word[j] + 1];
      s_shift128[j] = w128;
      w128 += bit_width_dev(hi - lo);
    }
    s_w128 = w128;
    // width of the leading key word inside the composite (word 0 comes last in the plan)
    s_keybits = (nwords > 0 && s_word[nwords - 1] == 0) ? w128 - s_shift128[nwords - 1] : 0;
    if (c == 0 && TW >= 0) a.kres[2] = n > 0 ? *(volatile u64*)&ctl->minmax[2 * (TW >= 0 ? TW : 0) + 1] : 0;
  }
  __syncthreads();
  const int nrounds = s_nrounds;
  PHASE_STAMP(1);
  if (a.dbg != nullptr && c == 0 && tid == 0) {
    a.dbg[16] = n;
    a.dbg[17] = (u64)nrounds;
    a.dbg[18] = (u64)(s_rbits[0] | ((u64)s_rbits[1] << 8) | ((u64)s_rbits[2] << 16) | ((u64)s_rbits[3] << 24));
    a.dbg[19] = G;
    a.dbg[20] = RB;
  }


  // =================================================================== MSD path
  bool msd_done = false;
  // (beyond ~256K rows the bucket phase stops paying: the look-back radix passes win)
  if (!merge && s_w128 <= 128 && n <= (a.fast != 0 ? MSD_FAST_MAX_ROWS : MSD_EXACT_MAX_ROWS)) {
    const int W = s_w128;
    auto composite = [&](const u64* row, u64* clo, u64* chi) {
      unsigned __int128 comp = 0;
      for (int j = 0; j < s_nwords; ++j)
        comp |= (unsigned __int128)(row[s_word[j]] - s_minv[j]) << s_shift128[j];
      *clo = (u64)comp;
      *chi = (u64)(comp >> 64);
    };
    auto bucket_of = [&](u64 clo, u64 chi) -> u32 {
      if (bb == 0 || W == 0) return 0u;
      const u64 top = W <= 64 ? (clo << (64 - W)) : ((chi << (128 - W)) | (W == 128 ? 0ull : (clo >> (W - 64))));
      return (u32)(top >> (64 - bb));
    };
    // ---- fast path: pack composites and scatter them straight into fixed-capacity bucket
    // regions (slot = the bucket's atomic counter), then one warp per bucket.  Two grid barriers
    // in all (after min/max, after the scatter); a bucket that outgrows its region (clumped
    // keys) raises ctl->overflow and the exact count -> scan -> scatter path below runs instead.
    bool fast_done = false, index_done = false;
    if (a.fast != 0) {
      const int Wr = W > (int)bb ? W - (int)bb : 0;  // bits that vary inside a bucket
      const bool narrow = Wr <= 64;
      // a key never spans two buckets when the bucket bits are all key bits
      const bool inline_index = a.table != nullptr && s_keybits >= (int)bb;
      for (u64 i = gtid; i < n; i += gstride) {
        u64 row[NW];
        load_in(i, row);
        u64 clo, chi;
        composite(row, &clo, &chi);
        const u32 b = bucket_of(clo, chi);
        const u32 r = atomicAdd(&ctl->bcnt[b], 1u);
        if (r < WCAP) {
          const u64 p = (u64)b * WCAP + r;
          if (narrow) {
            a.m_lo[p] = Wr >= 64 ? clo : (clo & ((1ull << Wr) - 1));
          } else {
            a.m_lo[p] = clo;
            a.m_hi[p] = Wr >= 128 ? chi : (chi & ((1ull << (Wr - 64)) - 1));
          }
          a.m_idx[p] = (u32)i;
        } else {
          *(volatile u32*)&ctl->overflow = 1u;
        }
      }
      if (inline_index)
        for (u64 i = gtid; i < (mask + 1) * 2; i += gstride) ((u64*)a.table)[i] = 0;
      grid_barrier(&ctl->barrier, G, epoch);
      PHASE_STAMP(10);
      if (*(volatile u32*)&ctl->overflow == 0u) {
        __shared__ u64 s_wcnt2[FT / 32 + 1];
        __shared__ u64 s_wlb2;
        __shared__ u32 s_stat2[2];
        if (tid == 0) {
          s_stat2[0] = 0;
          s_stat2[1] = 0;
        }
        __syncthreads();
        if (a.dbg != nullptr && c == 0 && tid == 0) {
          a.dbg[21] = narrow ? 4 : 5;
          a.dbg[22] = inline_index ? 1 : 0;
          a.dbg[23] = NB;
        }
        if (narrow)
          msd_warp_buckets2<RB, WR, 1>(a, ctl, NB, c, G, na, since, mask, inline_index, s_wcnt2, &s_wlb2,
                                       &sm.wkeys[0][0], s_stat2);
        else
          msd_warp_buckets2<RB, WR, 2>(a, ctl, NB, c, G, na, since, mask, inline_index, s_wcnt2, &s_wlb2,
                                       &sm.wkeys[0][0], s_stat2);
        fast_done = true;
        msd_done = true;
        index_done = inline_index;
      } else {
        for (u64 i = gtid; i < (u64)NB; i += gstride) ctl->bcnt[i] = 0;
        grid_barrier(&ctl->barrier, G, epoch);
      }
    }
    // the exact path keeps its bucket bases in shared memory: at most MSD_MAX_BUCKETS of them
    // (a bigger job whose fast path overflowed takes the radix path below)
    if (!fast_done && NB <= MSD_MAX_BUCKETS && n <= MSD_EXACT_MAX_ROWS) {
    // ---- pack composites, count rows per bucket (the atomic's return value is
    // the row's slot inside its bucket; the order inside a bucket is irrelevant)
    for (u64 i = gtid; i < n; i += gstride) {
      u64 row[NW];
      load_in(i, row);
      u64 clo, chi;
      composite(row, &clo, &chi);
      const u32 b = bucket_of(clo, chi);
      const u32 r = atomicAdd(&ctl->bcnt[b], 1u);
      a.k0[i] = clo;
      a.k1[i] = chi;
      a.v0[i] = r;
      a.v1[i] = b;
    }
    grid_barrier(&ctl->barrier, G, epoch);
    PHASE_STAMP(10);
    // ---- bucket bases (every CTA scans the same counts), size check, scatter
    {
      const u32 per = (NB + FT - 1) / FT;  // consecutive buckets per thread
      u32 local[MSD_MAX_BUCKETS / FT];
      u32 sum = 0, mx = 0;
#pragma unroll
      for (u32 j = 0; j < MSD_MAX_BUCKETS / FT; ++j) {
        const u32 bi = tid * per + j;
        u32 v = (j < per && bi < NB) ? *(volatile u32*)&ctl->bcnt[bi] : 0u;
        local[j] = v;
        sum += v;
        mx = v > mx ? v : mx;
      }
      if (tid == 0) s_max_bucket = 0;
      __syncthreads();
      atomicMax(&s_max_bucket, mx);
      u32 total;
      u32 ex = block_exclusive_scan(sum, sm_scan, &total);
#pragma unroll
      for (u32 j = 0; j < MSD_MAX_BUCKETS / FT; ++j) {
        const u32 bi = tid * per + j;
        if (j < per && bi < NB) {
          sm.scan.base[bi] = ex;
          ex += local[j];
        }
      }
      if (tid == 0) {
        sm.scan.base[NB] = total;
        s_max_unit = 0;
      }
      __syncthreads();
      // the CTA-level fallback works on units of eight consecutive buckets
      u32 mu = 0;
      for (u32 u = tid; u < (NB + 7) / 8; u += FT) {
        const u32 hi_b = (u * 8 + 8 < NB) ? u * 8 + 8 : NB;
        const u32 sz = sm.scan.base[hi_b] - sm.scan.base[u * 8];
        mu = sz > mu ? sz : mu;
      }
      atomicMax(&s_max_unit, mu);
      __syncthreads();
    }
    const u32 NU = (NB + 7) / 8;
    constexpr u32 LOCAL_MAX = ND == 8 ? 256u : MSD_LOCAL_MAX;
    if (a.dbg != nullptr && c == 0 && tid == 0) {
      a.dbg[21] = s_max_bucket <= WCAP ? 1 : (ND <= 8 && s_max_unit <= LOCAL_MAX ? 2 : 3);
      a.dbg[22] = s_max_bucket;
      a.dbg[23] = NB;
    }
    if (s_max_bucket <= WCAP) {
      // every bucket fits a warp.  Unreachable while fused_prepare sets `fast`: this exact path then
      // runs only after the fast path overflowed, i.e. some bucket of the same NB buckets held more
      // than WCAP rows, and the recount above finds that bucket again.
      for (u64 i = gtid; i < n; i += gstride) {
        const u64 p = (u64)sm.scan.base[a.v1[i]] + a.v0[i];
        a.m_lo[p] = a.k0[i];
        a.m_hi[p] = a.k1[i];
        a.m_idx[p] = (u32)i;
      }
      grid_barrier(&ctl->barrier, G, epoch);
      PHASE_STAMP(11);
      __shared__ u64 s_wcnt[FT / 32 + 1];
      __shared__ u64 s_wlb;
      msd_warp_buckets<RB, WR>(a, ctl, sm.scan.base, NB, c, G, na, since, s_wcnt, &s_wlb);
      msd_done = true;
    } else if (ND <= 8 && s_max_unit <= LOCAL_MAX) {  // (its shared sums hold at most 8 diff words)
      for (u64 i = gtid; i < n; i += gstride) {
        const u64 p = (u64)sm.scan.base[a.v1[i]] + a.v0[i];
        a.m_lo[p] = a.k0[i];
        a.m_hi[p] = a.k1[i];
        a.m_idx[p] = (u32)i;
      }
      grid_barrier(&ctl->barrier, G, epoch);
      PHASE_STAMP(11);
      // ---- per bucket: sort in shared memory, consolidate, emit
      const u64 upper = a.upper;
      LookBack lbs;
      lbs.state = a.lb_ship;
      lbs.ticket = nullptr;
      lbs.epoch = 1;
      __shared__ u64 s_lb;
      // this CTA's buckets (the bases live in the same shared memory as the sort arrays)
      u32 my_base[MSD_MAX_BUCKETS / 64 + 1], my_m[MSD_MAX_BUCKETS / 64 + 1];
      {
        int q = 0;
        for (u32 b = c; b < NU && q < (int)(MSD_MAX_BUCKETS / 64 + 1); b += G, ++q) {
          const u32 hi_b = (b * 8 + 8 < NB) ? b * 8 + 8 : NB;
          my_base[q] = sm.scan.base[b * 8];
          my_m[q] = sm.scan.base[hi_b] - sm.scan.base[b * 8];
        }
      }
      int q = 0;
      for (u32 b = c; b < NU; b += G, ++q) {  // b: unit of eight buckets
        const u32 gbase = my_base[q];
        const u32 m = my_m[q];
        u32 P = 32;
        while (P < m) P <<= 1;
        __syncthreads();
        for (u32 j = tid; j < P; j += FT) {
          if (j < m) {
            sm.msd.lo[j] = a.m_lo[gbase + j];
            sm.msd.hi[j] = a.m_hi[gbase + j];
            sm.msd.idx[j] = a.m_idx[gbase + j];
          } else {
            sm.msd.lo[j] = ~0ull;
            sm.msd.hi[j] = ~0ull;
            sm.msd.idx[j] = 0xffffffffu;
          }
          sm.msd.sum[j] = 0;
          if (ND == 8 && j < 256) {
#pragma unroll
            for (int w = 0; w < 8; ++w) sm.msd.sum8[j][w] = 0;
          }
        }
        __syncthreads();
        // bitonic sort of P elements by (hi, lo, idx); padding (all ones) sorts last
        for (u32 k = 2; k <= P; k <<= 1) {
          for (u32 j = k >> 1; j > 0; j >>= 1) {
            for (u32 i = tid; i < P; i += FT) {
              const u32 x = i ^ j;
              if (x > i) {
                const u64 hi1 = sm.msd.hi[i], lo1 = sm.msd.lo[i], hi2 = sm.msd.hi[x], lo2 = sm.msd.lo[x];
                const u32 i1 = sm.msd.idx[i], i2 = sm.msd.idx[x];
                const bool gt = hi1 > hi2 || (hi1 == hi2 && (lo1 > lo2 || (lo1 == lo2 && i1 > i2)));
                const bool up = (i & k) == 0;
                if (gt == up) {
                  sm.msd.hi[i] = hi2;
                  sm.msd.lo[i] = lo2;
                  sm.msd.idx[i] = i2;
                  sm.msd.hi[x] = hi1;
                  sm.msd.lo[x] = lo1;
                  sm.msd.idx[x] = i1;
                }
              }
            }
            __syncthreads();
          }
        }
        // pass 1: segmented diff sums over the sorted bucket.  Segment s of the bucket
        // accumulates in shared memory (one-word diffs) or in seg_sums[gbase + s].
        u32 nseg = 0;
        for (u32 j0 = 0; j0 < m; j0 += FT) {
          const u32 j = j0 + tid;
          const bool valid = j < m;
          u32 flag = 0;
          if (valid)
            flag = (j == 0 || sm.msd.lo[j] != sm.msd.lo[j - 1] || sm.msd.hi[j] != sm.msd.hi[j - 1]) ? 1u : 0u;
          u32 total;
          const u32 ex = block_exclusive_scan(flag, sm_scan, &total);
          const u32 seg = valid ? nseg + ex + flag - 1 : 0xffffffffu;
          u64 d[ND];
          if (valid) {
            u64 row[NW];
            load_in(sm.msd.idx[j], row);
#pragma unroll
            for (int w = 0; w < ND; ++w) d[w] = row[NK + w];
          } else {
#pragma unroll
            for (int w = 0; w < ND; ++w) d[w] = 0;
          }
          const u32 lane = lane_id();
#pragma unroll
          for (int off = 1; off < 32; off <<= 1) {
            u32 oseg = __shfl_up_sync(0xffffffffu, seg, off);
            u64 o[ND];
#pragma unroll
            for (int w = 0; w < ND; ++w) o[w] = __shfl_up_sync(0xffffffffu, d[w], off);
            if (lane >= (u32)off && oseg == seg) diff_add<ND>(d, o);
          }
          const u32 nxt = __shfl_down_sync(0xffffffffu, seg, 1);
          if (valid && (lane == 31 || nxt != seg)) {
            if (ND == 8) {
              u64* acc = &sm.msd.sum8[seg][0];
              if (d[0]) atomicAdd((unsigned long long*)&acc[0], (unsigned long long)d[0]);
              if (d[1]) atomicAdd((unsigned long long*)&acc[1], (unsigned long long)d[1]);
              u64 old = atomicAdd((unsigned long long*)&acc[2], (unsigned long long)d[2]);
              u64 hi = d[3] + ((old + d[2]) < old ? 1 : 0);
              if (hi) atomicAdd((unsigned long long*)&acc[3], (unsigned long long)hi);
              if (d[4]) atomicAdd((unsigned long long*)&acc[4], (unsigned long long)d[4]);
              if (d[5]) atomicAdd((unsigned long long*)&acc[5], (unsigned long long)d[5]);
              if (d[6]) atomicAdd((unsigned long long*)&acc[6], (unsigned long long)d[6]);
            } else {
              atomicAdd((unsigned long long*)&sm.msd.sum[seg], (unsigned long long)d[0]);
            }
          }
          nseg += total;
        }
        __syncthreads();
        // pass 2 (run twice: count, then write after the bucket-ordered look-back):
        // the head row of every surviving segment goes to `out` (time < upper) or `keep`
        u64 bases = 0;  // (ship << 21) | keep: exclusive prefix over earlier buckets
        u32 tot_ship = 0, tot_keep = 0;
        for (int pass = 0; pass < 2; ++pass) {
          u32 run_ship = 0, run_keep = 0, seg0 = 0;
          for (u32 j0 = 0; j0 < m; j0 += FT) {
            const u32 j = j0 + tid;
            const bool valid = j < m;
            u32 flag = 0;
            if (valid)
              flag = (j == 0 || sm.msd.lo[j] != sm.msd.lo[j - 1] || sm.msd.hi[j] != sm.msd.hi[j - 1]) ? 1u : 0u;
            u32 total;
            const u32 ex = block_exclusive_scan(flag, sm_scan, &total);
            u32 cls = 0;
            u64 r[NW];
            if (valid && flag) {
              const u32 seg = seg0 + ex;
              u64 d[ND];
              if (ND == 8) {
#pragma unroll
                for (int w = 0; w < ND; ++w) d[w] = sm.msd.sum8[seg][w & 7];
              } else {
                d[0] = sm.msd.sum[seg];
#pragma unroll
                for (int w = 1; w < ND; ++w) d[w] = 0;
              }
              if (!diff_is_zero<ND>(d)) {
                load_in(sm.msd.idx[j], r);
#pragma unroll
                for (int w = 0; w < ND; ++w) r[NK + w] = d[w];
                cls = (TW < 0 || upper == MZGPU_FRONTIER_EMPTY || r[TW >= 0 ? TW : 0] < upper) ? 1u : 2u;
              }
            }
            u32 t1, t2;
            const u32 e1 = block_exclusive_scan(cls == 1u ? 1u : 0u, sm_scan, &t1);
            const u32 e2 = block_exclusive_scan(cls == 2u ? 1u : 0u, sm_scan, &t2);
            if (pass == 1 && cls != 0u) {
              if (cls == 1u) {
                store_row<NW>(a.out, (bases >> 21) + run_ship + e1, r);
              } else if (a.keep != nullptr) {
                store_row<NW>(a.keep, (bases & ((1ull << 21) - 1)) + run_keep + e2, r);
                if (TW >= 0) atomicMin((unsigned long long*)&a.kres[1], (unsigned long long)r[TW >= 0 ? TW : 0]);
              }
            }
            run_ship += t1;
            run_keep += t2;
            seg0 += total;
          }
          if (pass == 0) {
            tot_ship = run_ship;
            tot_keep = run_keep;
            bases = lb_exclusive_prefix(lbs, b, ((u64)tot_ship << 21) | (u64)tot_keep, &s_lb);
          }
        }
        if (b == NU - 1 && tid == 0) {
          ctl->n_out = (bases >> 21) + tot_ship;
          a.res[0] = (bases >> 21) + tot_ship;
          a.kres[0] = (bases & ((1ull << 21) - 1)) + tot_keep;
        }
      }
      msd_done = true;
    }
    }  // !fast_done
    if (index_done) {
      PHASE_STAMP(7);
      return;
    }
  }
  PHASE_STAMP(7);
  if (msd_done) {
    if (a.table == nullptr) return;
    // the table is cleared here, off the critical path of the earlier phases (CTAs
    // reach this point at different times; the index is built after the barrier)
    for (u64 i = gtid; i < (mask + 1) * 2; i += gstride) ((u64*)a.table)[i] = 0;
    grid_barrier(&ctl->barrier, G, epoch);
    PHASE_STAMP(8);
  }
  u64 n_out = 0;
  if (!msd_done) {
  const u64 U = (n + FT - 1) / FT;
  auto is_head = [&](u64 i) -> u32 {
    if (i == 0) return 1u;
    const u64* p = a.sorted + i * NW;
#pragma unroll
    for (int k = 0; k < NK; ++k)
      if (p[k] != p[k - NW]) return 1u;
    return 0u;
  };
  // the sort / merge paths accumulate segment sums in global memory (used several
  // grid barriers from here)
  for (u64 i = gtid; i < n * ND; i += gstride) a.seg_sums[i] = 0;
  if (!merge) {
  // ---- radix rounds.  (kin, vin) holds the current order; round r packs into the
  // other pair (reading the order of round r-1) and sorts that.
  u64* kcur = a.k0;
  u32* vcur = a.v0;
  u64* kalt = a.k1;
  u32* valt = a.v1;
  u32 gpass = 0;  // passes done so far (selects the look-back state buffer)
  if (nrounds == 0) {
    for (u64 i = gtid; i < n; i += gstride) {
      kcur[i] = 0;
      vcur[i] = (u32)i;
    }
    grid_barrier(&ctl->barrier, G, epoch);
  }
  for (int r = 0; r < nrounds; ++r) {
    const int npass = (s_rbits[r] + 7) / 8;
    u32* hist = ctl->hist + r * 8 * 256;
    // pack + histogram of every digit place of this round
    for (int i = tid; i < 8 * 256; i += FT) sm.hist[i] = 0;
    __syncthreads();
    u64* kdst = r == 0 ? kcur : kalt;
    u32* vdst = r == 0 ? vcur : valt;
    for (u64 i = gtid; i < n; i += gstride) {
      const u32 src = r == 0 ? (u32)i : vcur[i];
      u64 row[NW];
      load_in(src, row);
      u64 comp = 0;
      for (int j = 0; j < s_nwords; ++j)
        if (s_round[j] == r) comp |= (row[s_word[j]] - s_minv[j]) << s_shift[j];
      kdst[i] = comp;
      vdst[i] = src;
      for (int ps = 0; ps < npass; ++ps) atomicAdd(&sm.hist[ps * 256 + (u32)((comp >> (8 * ps)) & 255)], 1u);
    }
    __syncthreads();
    for (int i = tid; i < npass * 256; i += FT) {
      u32 v = sm.hist[i];
      if (v) atomicAdd(&hist[i], v);
    }
    if (r > 0) {
      u64* tk = kcur;
      kcur = kalt;
      kalt = tk;
      u32* tv = vcur;
      vcur = valt;
      valt = tv;
    }
    grid_barrier(&ctl->barrier, G, epoch);
    // exclusive scan of each pass's histogram (one CTA per pass)
    for (int ps = c; ps < npass; ps += G) {
      u32 v = *(volatile u32*)&hist[ps * 256 + tid];
      u32 total;
      u32 ex = block_exclusive_scan(v, sm_scan, &total);
      hist[ps * 256 + tid] = ex;
    }
    grid_barrier(&ctl->barrier, G, epoch);
    // passes.  CTA c takes tiles c, c+G, ...: every predecessor of a tile is done
    // or in flight on a co-resident CTA.  The other state buffer is cleared for
    // the next pass meanwhile.
    for (int ps = 0; ps < npass; ++ps, ++gpass) {
      u32* st = (gpass & 1) ? a.state1 : a.state0;
      u32* st_next = (gpass & 1) ? a.state0 : a.state1;
      for (u64 t = c; t < T; t += G) {
        for (int i = tid; i < 256; i += FT) st_next[t * 256 + i] = 0;
        rs_tile_pass<FI>(sm.rs, (u32)t, kcur, vcur, kalt, valt, n, 8 * ps, hist + ps * 256, st);
      }
      grid_barrier(&ctl->barrier, G, epoch);
      u64* tk = kcur;
      kcur = kalt;
      kalt = tk;
      u32* tv = vcur;
      vcur = valt;
      valt = tv;
    }
  }
  const u32* perm = vcur;  // final order
  PHASE_STAMP(2);
  // ---- gather rows by the final permutation
  for (u64 u = c; u < U; u += G) {
    const u64 i = u * FT + tid;
    if (i < n) {
      u64 r[NW];
      load_in(perm[i], r);
      store_row<NW>(a.sorted, i, r);
    }
  }
  } else {
    // ---- merge path: A and B are sorted (and stay sorted under advance_by(since),
    // which is monotone); every thread finds its diagonal by binary search and
    // merges MV consecutive outputs.  Ties take A first (A is the older batch).
    constexpr int MV = 4;
    auto less_ba = [&](const u64* x, const u64* y) -> bool {  // x < y on the key words, times advanced
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        u64 p = x[k], q = y[k];
        if (k == TW) {
          p = p < since ? since : p;
          q = q < since ? since : q;
        }
        if (p != q) return p < q;
      }
      return false;
    };
    const u64 n_groups = (n + (u64)FT * MV - 1) / ((u64)FT * MV);
    __shared__ u32 s_tc[MV];
    auto keys_differ = [&](const u64* x, const u64* y) -> bool {
#pragma unroll
      for (int k = 0; k < NK; ++k)
        if (x[k] != y[k]) return true;
      return false;
    };
    for (u64 u = c; u < n_groups; u += G) {
      const u64 o0 = (u * FT + tid) * MV;
      __syncthreads();
      if (tid < MV) s_tc[tid] = 0;
      __syncthreads();
      u32 heads = 0;
      if (o0 < n) {
        u64 lo = o0 > nb ? o0 - nb : 0, hi = o0 < na ? o0 : na;
        while (lo < hi) {
          const u64 mid = (lo + hi) >> 1;
          const u64 bi = o0 - mid;  // >= 1
          if (!less_ba(a.b + (bi - 1) * NW, a.a + mid * NW))
            lo = mid + 1;
          else
            hi = mid;
        }
        u64 ia = lo, ib = o0 - lo;
        // the output just before mine (ties put the B row later), times advanced
        u64 prev[NW];
        bool have_prev = o0 > 0;
        if (have_prev) {
          const bool use_b = ib > 0 && (ia == 0 || !less_ba(a.b + (ib - 1) * NW, a.a + (ia - 1) * NW));
          if (use_b)
            load_row<NW>(a.b, ib - 1, prev);
          else
            load_row<NW>(a.a, ia - 1, prev);
          if (TW >= 0) {
            u64& t = prev[TW >= 0 ? TW : 0];
            t = t < since ? since : t;
          }
        }
#pragma unroll
        for (int k = 0; k < MV; ++k) {
          const u64 o = o0 + k;
          if (o >= n) break;
          const bool take_a = ib >= nb || (ia < na && !less_ba(a.b + ib * NW, a.a + ia * NW));
          u64 r[NW];
          if (take_a)
            load_row<NW>(a.a, ia++, r);
          else
            load_row<NW>(a.b, ib++, r);
          if (TW >= 0) {
            u64& t = r[TW >= 0 ? TW : 0];
            t = t < since ? since : t;
          }
          store_row<NW>(a.sorted, o, r);
          if (!have_prev || keys_differ(r, prev)) ++heads;
          have_prev = true;
#pragma unroll
          for (int w = 0; w < NW; ++w) prev[w] = r[w];
        }
      }
      // head counts of the 256-row tiles of this group (64 threads each)
      if (heads) atomicAdd(&s_tc[tid / (FT / MV)], heads);
      __syncthreads();
      if (tid < MV) {
        const u64 tile = u * MV + tid;
        if (tile < U) a.tile_cnt[tile] = s_tc[tid];
      }
    }
  }
  grid_barrier(&ctl->barrier, G, epoch);
  PHASE_STAMP(3);
  if (!merge) {  // (the merge phase has already counted the heads of every tile)
    for (u64 u = c; u < U; u += G) {
      const u64 i = u * FT + tid;
      u32 flag = i < n ? is_head(i) : 0u;
      u32 total;
      block_exclusive_scan(flag, sm_scan, &total);
      if (tid == 0) a.tile_cnt[u] = total;
    }
    grid_barrier(&ctl->barrier, G, epoch);
  }

  PHASE_STAMP(4);
  // ---- segmented sums
  for (u64 u = c; u < U; u += G) {
    const u32 base = block_sum_prefix(a.tile_cnt, u, sm_scan);
    const u64 i = u * FT + tid;
    const bool valid = i < n;
    u32 flag = valid ? is_head(i) : 0u;
    u32 total;
    u32 ex = block_exclusive_scan(flag, sm_scan, &total);
    u32 seg = valid ? base + ex + flag - 1 : 0xffffffffu;
    u64 d[ND];
#pragma unroll
    for (int w = 0; w < ND; ++w) d[w] = valid ? a.sorted[i * NW + NK + w] : 0;
    if (valid && flag) a.seg_first[seg] = (u32)i;
    const u32 lane = lane_id();
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      u32 oseg = __shfl_up_sync(0xffffffffu, seg, off);
      u64 o[ND];
#pragma unroll
      for (int w = 0; w < ND; ++w) o[w] = __shfl_up_sync(0xffffffffu, d[w], off);
      if (lane >= (u32)off && oseg == seg) diff_add<ND>(d, o);
    }
    u32 nseg = __shfl_down_sync(0xffffffffu, seg, 1);
    if (valid && (lane == 31 || nseg != seg)) {
      u64* acc = a.seg_sums + (u64)seg * ND;
      if (ND == 8) {
        if (d[0]) atomicAdd((unsigned long long*)&acc[0], (unsigned long long)d[0]);
        if (d[1]) atomicAdd((unsigned long long*)&acc[1], (unsigned long long)d[1]);
        u64 old = atomicAdd((unsigned long long*)&acc[2], (unsigned long long)d[2]);
        u64 hi = d[3] + ((old + d[2]) < old ? 1 : 0);
        if (hi) atomicAdd((unsigned long long*)&acc[3], (unsigned long long)hi);
        if (d[4]) atomicAdd((unsigned long long*)&acc[4], (unsigned long long)d[4]);
        if (d[5]) atomicAdd((unsigned long long*)&acc[5], (unsigned long long)d[5]);
        if (d[6]) atomicAdd((unsigned long long*)&acc[6], (unsigned long long)d[6]);
      } else if (ND > 8) {
        atomic_lanes_add<ND>(acc, d);
      } else {
        atomicAdd((unsigned long long*)&acc[0], (unsigned long long)d[0]);
      }
    }
    if (u == U - 1 && tid == 0) ctl->n_seg = (u64)base + total;
  }
  grid_barrier(&ctl->barrier, G, epoch);

  PHASE_STAMP(5);
  // ---- surviving segments per tile: ship (time < upper) and keep
  const u64 S = U == 0 ? 0 : *(volatile u64*)&ctl->n_seg;
  const u64 V = (S + FT - 1) / FT;
  const u64 upper = a.upper;
  auto seg_class = [&](u64 s, u64* d) -> u32 {  // 0 dropped, 1 ship, 2 keep
#pragma unroll
    for (int w = 0; w < ND; ++w) d[w] = *(volatile u64*)&a.seg_sums[s * ND + w];
    if (diff_is_zero<ND>(d)) return 0u;
    if (TW < 0 || upper == MZGPU_FRONTIER_EMPTY) return 1u;
    const u64 t = a.sorted[(u64)a.seg_first[s] * NW + (TW >= 0 ? TW : 0)];
    return t < upper ? 1u : 2u;
  };
  for (u64 v = c; v < V; v += G) {
    const u64 s = v * FT + tid;
    u64 d[ND];
    u32 cls = s < S ? seg_class(s, d) : 0u;
    u32 total;
    block_exclusive_scan(cls == 1u ? 1u : 0u, sm_scan, &total);
    if (tid == 0) a.tile_cnt[v] = total;
    block_exclusive_scan(cls == 2u ? 1u : 0u, sm_scan, &total);
    if (tid == 0) a.tile_cnt2[v] = total;
  }
  grid_barrier(&ctl->barrier, G, epoch);

  PHASE_STAMP(6);
  // ---- emit
  for (u64 v = c; v < V; v += G) {
    const u32 base = block_sum_prefix(a.tile_cnt, v, sm_scan);
    const u32 base2 = a.keep != nullptr ? block_sum_prefix(a.tile_cnt2, v, sm_scan) : 0u;
    const u64 s = v * FT + tid;
    u64 d[ND];
    u32 cls = s < S ? seg_class(s, d) : 0u;
    u32 total, total2;
    u32 ex = block_exclusive_scan(cls == 1u ? 1u : 0u, sm_scan, &total);
    u32 ex2 = block_exclusive_scan(cls == 2u ? 1u : 0u, sm_scan, &total2);
    if (cls != 0u) {
      u64 r[NW];
      load_row<NW>(a.sorted, a.seg_first[s], r);
#pragma unroll
      for (int w = 0; w < ND; ++w) r[NK + w] = d[w];
      if (cls == 1u) {
        store_row<NW>(a.out, (u64)base + ex, r);
      } else if (a.keep != nullptr) {
        store_row<NW>(a.keep, (u64)base2 + ex2, r);
        if (TW >= 0) atomicMin((unsigned long long*)&a.kres[1], (unsigned long long)r[TW >= 0 ? TW : 0]);
      }
    }
    if (v == V - 1 && tid == 0) {
      ctl->n_out = (u64)base + total;
      a.res[0] = (u64)base + total;
      a.kres[0] = (u64)base2 + total2;
    }
  }
  PHASE_STAMP(7);
  if (a.table == nullptr) return;
  for (u64 i = gtid; i < (mask + 1) * 2; i += gstride) ((u64*)a.table)[i] = 0;
  grid_barrier(&ctl->barrier, G, epoch);
  PHASE_STAMP(8);
  n_out = V == 0 ? 0 : *(volatile u64*)&ctl->n_out;
  } else {
    n_out = *(volatile u64*)&ctl->n_out;
  }

  // ---- hash index over the distinct keys of the output; longest key run
  // (key count and longest run are reduced per CTA: one global atomic each)
  __shared__ u32 s_nheads, s_runmax;
  if (tid == 0) {
    s_nheads = 0;
    s_runmax = 0;
  }
  __syncthreads();
  u32 my_run = 0, my_heads = 0;
  for (u64 i = gtid; i < ((n_out + 31) / 32) * 32; i += gstride) {
    bool head = false;
    u64 key = 0;
    if (i < n_out) {
      key = a.out[i * NW];
      head = (i == 0) || a.out[(i - 1) * NW] != key;
    }
    u32 m = __ballot_sync(0xffffffffu, head);
    my_heads += __popc(m);
    if (head) {
      u32 run = 1;
      while (run < MAX_RUN_SAT && i + run < n_out && a.out[(i + run) * NW] == key) ++run;
      my_run = run > my_run ? run : my_run;
      // slot: first row + 1, and the run length when it did not saturate
      const u64 meta = (i + 1) | ((u64)(run < MAX_RUN_SAT ? run : 0u) << 44);
      u64 h = mix64(key) & mask;
      while (true) {
        unsigned long long prev = atomicCAS((unsigned long long*)&a.table[h].meta, 0ull, (unsigned long long)meta);
        if (prev == 0ull) {
          a.table[h].key = key;
          break;
        }
        h = (h + 1) & mask;
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    u32 o = __shfl_xor_sync(0xffffffffu, my_run, off);
    my_run = o > my_run ? o : my_run;
  }
  if (lane_id() == 0) {
    if (my_heads) atomicAdd(&s_nheads, my_heads);
    if (my_run) atomicMax(&s_runmax, my_run);
  }
  __syncthreads();
  if (tid == 0) {
    if (s_nheads) atomicAdd((unsigned long long*)&a.res[2], (unsigned long long)s_nheads);
    if (s_runmax) atomicMax((unsigned long long*)&a.res[3], (unsigned long long)s_runmax);
  }
  PHASE_STAMP(9);
}

template <int RB>
__global__ void __launch_bounds__(FT, (RB >= 80 ? 2 : 4)) k_fused_consolidate(const FusedArgs a) {
  fused_body<RB>(a, blockIdx.x, gridDim.x);
}

// Several independent jobs of one row width in ONE cooperative launch (the arrangement seals of
// one timestamp, the merges their inserts trigger): job j owns CTAs [start[j], start[j+1]).  An
// update-batch job is a chain of latency-bound phases that leaves most of the machine idle, so
// jobs side by side cost about as much as the longest of them alone.
constexpr int FUSED_MANY_MAX = MZ_FUSED_MANY_MAX;
struct FusedMany {
  u32 k;
  u32 start[FUSED_MANY_MAX + 1];
  FusedArgs job[FUSED_MANY_MAX];
};
template <int RB>
__global__ void __launch_bounds__(FT, (RB >= 80 ? 2 : 4)) k_fused_many(const __grid_constant__ FusedMany m) {
  u32 j = 0;
  while (j + 1 < m.k && blockIdx.x >= m.start[j + 1]) ++j;
  fused_body<RB>(m.job[j], blockIdx.x - m.start[j], m.start[j + 1] - m.start[j]);
}

// Two sorted update-batch-sized inputs merge faster as a sort of A ++ B on the fast MSD path; from a few
// hundred thousand rows each the merge-path form wins.
constexpr u32 MERGE_SORT_MAX = 1u << 18;

// Everything of a launch but the launch: buffers, control block, kernel arguments.
// `slot` < 0: the context's single-job control blocks; otherwise job slot `slot` of a
// multi-job launch (each slot flips between its own pair of control blocks).
template <int RB>
int32_t fused_prepare(mzgpu_ctx* ctx, const FusedJob& job, FusedOut* res, int slot, FusedArgs* a_out,
                      u64* want_out, DevMem* scratch) {
  constexpr int ND = RowT<RB>::ND;
  const u64 cap = job.cap > 0 ? job.cap : 1;
  if (cap > MZ_FUSED_MAX_CAP) {
    MZ_SET_ERR(ctx, "fused consolidate: %llu rows exceed the fused limit", (unsigned long long)cap);
    return MZGPU_E_INVALID;
  }
  FusedArgs& a = *a_out;
  memset(&a, 0, sizeof(a));
  a.a = (const u64*)job.a;
  a.b = (const u64*)job.b;
  a.na = job.na;
  a.nb = job.nb;
  a.since = job.since;
  a.upper = job.upper;
  const u64 Tcap = (cap + FTILE - 1) / FTILE;
  const u64 Ucap = (cap + FT - 1) / FT;
  u64 slots = 0;
  if (job.want_index) {
    slots = 2;
    while (slots < 2 * cap) slots <<= 1;
  }
  // one scratch allocation, carved up (every region 16-byte aligned)
  auto al = [](u64 x) { return (x + 15) & ~(u64)15; };
  const u64 o_k0 = 0, o_k1 = o_k0 + al(cap * 8), o_v0 = o_k1 + al(cap * 8), o_v1 = o_v0 + al(cap * 4);
  const u64 o_s0 = o_v1 + al(cap * 4), o_s1 = o_s0 + al(Tcap * 1024), o_sorted = o_s1 + al(Tcap * 1024);
  const u64 o_t1 = o_sorted + al(cap * RB), o_t2 = o_t1 + al(Ucap * 4), o_sums = o_t2 + al(Ucap * 4);
  // the fast MSD path's buckets are fixed-capacity regions (128 slots each): the bucket arrays
  // hold (buckets for the largest row count this launch can see) x 128 entries
  u64 mcap = cap;
  {
    const u64 n_max = cap < MSD_FAST_MAX_ROWS ? cap : MSD_FAST_MAX_ROWS;
    u32 bb = 0;
    while (bb < 15 && ((u64)(ND >= 8 ? 12 : 48) << bb) < n_max) ++bb;
    const u64 regions = ((u64)1 << bb) * 128;
    if (regions > mcap) mcap = regions;
  }
  const u64 o_first = o_sums + al(cap * ND * 8), o_mlo = o_first + al(cap * 4);
  const u64 o_mhi = o_mlo + al(mcap * 8), o_midx = o_mhi + al(mcap * 8), o_lbs = o_midx + al(mcap * 4);
  const u64 o_lbk = o_lbs + MSD_MAX_BUCKETS * 8, o_end = o_lbk + MSD_MAX_BUCKETS * 8;
  MZ_TRY(scratch->alloc(ctx, o_end));
  MZ_TRY(res->rows.alloc(ctx, cap * RB));
  res->rows_cap = cap;
  const bool want_keep = job.upper != MZGPU_FRONTIER_EMPTY && RowT<RB>::TW >= 0;
  if (want_keep) MZ_TRY(res->keep.alloc(ctx, cap * RB));
  if (job.want_index) MZ_TRY(res->table.alloc(ctx, slots * sizeof(HashSlot)));
  MZ_TRY(res->st.make_pending(ctx));
  MZ_TRY(res->kst.make_pending(ctx));
  char* sp = (char*)scratch->p;
  if (slot < 0) {
    const int si = (ctx->side_stream != nullptr && ctx->stream == ctx->side_stream) ? 1 : 0;
    a.ctl = (FusedCtl*)ctx->d_fused_ctl[2 * si + ctx->fused_flip[si]];
    a.ctl_next = (FusedCtl*)ctx->d_fused_ctl[2 * si + (ctx->fused_flip[si] ^ 1)];
    ctx->fused_flip[si] ^= 1;
  } else {
    a.ctl = (FusedCtl*)ctx->d_fused_ctl_many[2 * slot + ctx->fused_flip_many[slot]];
    a.ctl_next = (FusedCtl*)ctx->d_fused_ctl_many[2 * slot + (ctx->fused_flip_many[slot] ^ 1)];
    ctx->fused_flip_many[slot] ^= 1;
  }
  a.k0 = (u64*)(sp + o_k0);
  a.k1 = (u64*)(sp + o_k1);
  a.v0 = (u32*)(sp + o_v0);
  a.v1 = (u32*)(sp + o_v1);
  a.state0 = (u32*)(sp + o_s0);
  a.state1 = (u32*)(sp + o_s1);
  a.sorted = (u64*)(sp + o_sorted);
  a.tile_cnt = (u32*)(sp + o_t1);
  a.tile_cnt2 = (u32*)(sp + o_t2);
  a.seg_sums = (u64*)(sp + o_sums);
  a.seg_first = (u32*)(sp + o_first);
  a.m_lo = (u64*)(sp + o_mlo);
  a.m_hi = (u64*)(sp + o_mhi);
  a.m_idx = (u32*)(sp + o_midx);
  a.lb_ship = (u64*)(sp + o_lbs);
  a.lb_keep = (u64*)(sp + o_lbk);
  a.merge = (job.merge && job.b != nullptr) ? 1u : 0u;
  a.out = res->rows.template as<u64>();
  a.keep = want_keep ? res->keep.template as<u64>() : nullptr;
  a.table = job.want_index ? res->table.template as<HashSlot>() : nullptr;
  a.table_cap = slots;
  a.res = res->st.dptr();
  a.kres = res->kst.dptr();
  a.fast = 1u;
  a.merge_sort_max = MERGE_SORT_MAX;
  a.dbg = nullptr;
  if (ctx->profile && ctx->d_dbg != nullptr && ctx->dbg_next < MZ_DBG_RECORDS) {
    a.dbg = ctx->d_dbg + 32 * (size_t)ctx->dbg_next++;
    MZ_CUDA(ctx, cudaMemsetAsync(a.dbg, 0, 32 * 8, ctx->stream));
  }
  *want_out = (cap + 127) / 128 + 1;  // one CTA per MSD bucket (128..256 rows each), at least one per radix tile
  return MZGPU_OK;
}

template <int RB>
int32_t fused_t(mzgpu_ctx* ctx, const FusedJob& job, FusedOut* res) {
  static int max_ctas = 0;
  if (max_ctas == 0) {
    int per_sm = 0;
    MZ_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_fused_consolidate<RB>, FT, 0));
    max_ctas = per_sm * ctx->num_sms;
    if (max_ctas <= 0) {
      MZ_SET_ERR(ctx, "fused kernel cannot be made resident");
      return MZGPU_E_CUDA;
    }
  }
  FusedArgs a;
  u64 want = 0;
  DevMem scratch;
  MZ_TRY(fused_prepare<RB>(ctx, job, res, -1, &a, &want, &scratch));
  // A launch ON the side stream (a merge too large for the merge-path kernels' look-back state; the
  // ordinary spine merges there are plain launches, mergepath.cu) takes at most one CTA slot per SM, so
  // that it can be co-resident with the operators' launches on the main stream (a cooperative launch
  // starts when its whole grid fits).  Main-stream launches use the whole resident capacity:
  // (64 registers per thread: four CTAs per SM are resident, 528 on an H100; the bucket phase
  // wants one warp per bucket, and a 160K-row merge has 4096 of them)
  const bool on_side = ctx->side_stream != nullptr && ctx->stream == ctx->side_stream;
  a.max_g = on_side ? (u32)ctx->num_sms : (u32)max_ctas;
  if (a.max_g > (u32)max_ctas) a.max_g = (u32)max_ctas;
  const unsigned a_max_g_host = a.max_g;
  unsigned grid = (unsigned)(want < (u64)max_ctas ? want : (u64)max_ctas);
  if (grid > a_max_g_host) grid = a_max_g_host;
  if (grid == 0) grid = 1;
  void* kargs[] = {(void*)&a};
  {
    // algorithmic bytes: 4 x rows x row bytes (read for min/max, read to pack, read to gather/emit,
    // written out).  With a device-resident count only the bound is known here;
    // mzgpu_profile_report substitutes the actual row count of profiled launches.
    MZ_BYTES(ctx, (job.na.p == nullptr && job.nb.p == nullptr) ? (job.na.imm + job.nb.imm) * RB * 4 : 0);
    ProfScope prof(ctx, "k_fused_consolidate");
    const cudaError_t e =
        cudaLaunchCooperativeKernel((void*)k_fused_consolidate<RB>, dim3(grid), dim3(FT), kargs, 0, ctx->stream);
    if (e != cudaSuccess) {
      MZ_SET_ERR(ctx, "cooperative launch failed: %s", cudaGetErrorString(e));
      ctx->sticky = true;
      return MZGPU_E_CUDA;
    }
  }
  ctx->stats.kernel_launches++;
  res->st.mark_written();
  res->kst.mark_written();
  return MZGPU_OK;
}

// k prepared jobs (same row width) in one cooperative launch.  The resident capacity is
// shared out in proportion to what each job alone would take.
template <int RB>
int32_t fused_launch_many(mzgpu_ctx* ctx, int k, const FusedArgs* args, const u64* want_in, u64 bytes) {
  static int max_ctas = 0;
  if (max_ctas == 0) {
    int per_sm = 0;
    MZ_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_fused_many<RB>, FT, 0));
    max_ctas = per_sm * ctx->num_sms;
    if (max_ctas <= 0) {
      MZ_SET_ERR(ctx, "fused kernel cannot be made resident");
      return MZGPU_E_CUDA;
    }
  }
  static thread_local FusedMany m;  // ~1.5 KB, passed by value
  memset(&m, 0, sizeof(m));
  m.k = (u32)k;
  u64 want[FUSED_MANY_MAX];
  u64 want_sum = 0;
  const u64 solo_max = (u64)max_ctas;
  for (int j = 0; j < k; ++j) {
    m.job[j] = args[j];
    want[j] = want_in[j] > solo_max ? solo_max : want_in[j];
    if (want[j] == 0) want[j] = 1;
    want_sum += want[j];
  }
  u32 at = 0;
  for (int j = 0; j < k; ++j) {
    u64 g = want_sum <= (u64)max_ctas ? want[j] : want[j] * (u64)max_ctas / want_sum;
    if (g == 0) g = 1;
    m.start[j] = at;
    m.job[j].max_g = (u32)g;
    at += (u32)g;
  }
  m.start[k] = at;
  if ((int)at > max_ctas) {  // k jobs of one CTA each always fit: k <= FUSED_MANY_MAX << max_ctas
    MZ_SET_ERR(ctx, "fused multi-job launch: %u CTAs exceed the resident capacity %d", at, max_ctas);
    return MZGPU_E_INVALID;
  }
  void* kargs[] = {(void*)&m};
  {
    MZ_BYTES(ctx, bytes);
    ProfScope prof(ctx, "k_fused_consolidate");  // one profile line for the operator, whatever the launch shape
    const cudaError_t e =
        cudaLaunchCooperativeKernel((void*)k_fused_many<RB>, dim3(at), dim3(FT), kargs, 0, ctx->stream);
    if (e != cudaSuccess) {
      MZ_SET_ERR(ctx, "cooperative launch failed: %s", cudaGetErrorString(e));
      ctx->sticky = true;
      return MZGPU_E_CUDA;
    }
  }
  ctx->stats.kernel_launches++;
  return MZGPU_OK;
}

static u64 fused_job_bytes(const FusedJob& job) {
  return (job.na.p == nullptr && job.nb.p == nullptr) ? (job.na.imm + job.nb.imm) * (u64)job.rb * 4 : 0;
}

template <int RB>
int32_t fused_many_t(mzgpu_ctx* ctx, int k, const FusedJob* jobs, FusedOut* outs) {
  FusedArgs args[FUSED_MANY_MAX];
  DevMem scratch[FUSED_MANY_MAX];
  u64 want[FUSED_MANY_MAX];
  u64 bytes = 0;
  for (int j = 0; j < k; ++j) {
    MZ_TRY(fused_prepare<RB>(ctx, jobs[j], &outs[j], j, &args[j], &want[j], &scratch[j]));
    bytes += fused_job_bytes(jobs[j]);
  }
  MZ_TRY(fused_launch_many<RB>(ctx, k, args, want, bytes));
  for (int j = 0; j < k; ++j) {
    outs[j].st.mark_written();
    outs[j].kst.mark_written();
  }
  return MZGPU_OK;
}

// Jobs prepared now and launched together later (mz_fused_defer / mz_fused_flush): the merges that
// the spine inserts of one timestamp trigger.  Their control blocks are the job slots
// FUSED_MANY_MAX .. 2 * FUSED_MANY_MAX - 1, used in prepare order = launch order.
struct FusedDeferred {
  int rb = 0;
  int k = 0;
  FusedArgs args[FUSED_MANY_MAX];
  u64 want[FUSED_MANY_MAX];
  DevMem scratch[FUSED_MANY_MAX];
  u64 bytes = 0;
};

template <int RB>
int32_t fused_defer_t(mzgpu_ctx* ctx, FusedDeferred* d, const FusedJob& job, FusedOut* out) {
  const int j = d->k;
  MZ_TRY(fused_prepare<RB>(ctx, job, out, FUSED_MANY_MAX + j, &d->args[j], &d->want[j], &d->scratch[j]));
  d->bytes += fused_job_bytes(job);
  d->rb = RB;
  d->k = j + 1;
  return MZGPU_OK;
}

}  // namespace

size_t mz_fused_ctl_bytes() { return sizeof(FusedCtl); }

int32_t mz_fused_flush(mzgpu_ctx* ctx) {
  FusedDeferred* d = (FusedDeferred*)ctx->fused_deferred;
  if (d == nullptr || d->k == 0) return MZGPU_OK;
  const int k = d->k;
  d->k = 0;  // whatever happens below, the jobs are not retried
  ctx->deferred_unlaunched = 0;
  const int32_t st = mz_dispatch<RowWidths>(ctx, d->rb, "fused flush", [&](auto RB) {
    return fused_launch_many<RB>(ctx, k, d->args, d->want, d->bytes);
  });
  for (int j = 0; j < k; ++j) d->scratch[j].release();  // stream ordered: after the launch
  d->bytes = 0;
  mz_cnt_unpark(ctx);  // counter blocks freed while the jobs waited (their inputs' lengths)
  if (st != MZGPU_OK) ctx->sticky = true;  // outputs were promised to readers
  return st;
}

void mz_fused_deferred_free(mzgpu_ctx* ctx) {
  delete (FusedDeferred*)ctx->fused_deferred;
  ctx->fused_deferred = nullptr;
}

// Prepare `job` (buffers, counters, control block) and leave the launch to mz_fused_flush.  The
// result counters count as written from now on: mz_resolve_counters flushes before it copies the
// arena, so a counter can never be read back ahead of its launch.
int32_t mz_fused_defer(mzgpu_ctx* ctx, const FusedJob& job, FusedOut* out) {
  if (ctx->fused_deferred == nullptr) ctx->fused_deferred = new FusedDeferred();
  FusedDeferred* d = (FusedDeferred*)ctx->fused_deferred;
  if (d->k > 0 && (d->rb != job.rb || d->k == FUSED_MANY_MAX)) MZ_TRY(mz_fused_flush(ctx));
  MZ_TRY(mz_dispatch<RowWidths>(ctx, job.rb, "fused", [&](auto RB) { return fused_defer_t<RB>(ctx, d, job, out); }));
  ctx->deferred_unlaunched = d->k;
  out->st.mark_written();
  out->kst.mark_written();
  return MZGPU_OK;
}

int32_t mz_fused_consolidate_many(mzgpu_ctx* ctx, int k, const FusedJob* jobs, FusedOut* outs) {
  if (k <= 0) return MZGPU_OK;
  if (k == 1) return mz_fused_consolidate(ctx, jobs[0], &outs[0]);
  if (k > FUSED_MANY_MAX) {
    MZ_SET_ERR(ctx, "fused multi-job launch: %d jobs exceed the maximum %d", k, FUSED_MANY_MAX);
    return MZGPU_E_INVALID;
  }
  for (int j = 1; j < k; ++j)
    if (jobs[j].rb != jobs[0].rb) {
      MZ_SET_ERR(ctx, "fused multi-job launch: mixed row widths %d / %d", jobs[0].rb, jobs[j].rb);
      return MZGPU_E_INVALID;
    }
  return mz_dispatch<RowWidths>(ctx, jobs[0].rb, "fused", [&](auto RB) { return fused_many_t<RB>(ctx, k, jobs, outs); });
}

int32_t mz_fused_consolidate(mzgpu_ctx* ctx, const FusedJob& job, FusedOut* res) {
  return mz_dispatch<RowWidths>(ctx, job.rb, "fused", [&](auto RB) { return fused_t<RB>(ctx, job, res); });
}
