// mfp.cu — temporal filters: the device MfpPlan (include/mzgpu.h, mzgpu_mfp_new) and the partition
// kernels of the bucket chain that holds its future updates (host.cu: mzgpu_mfp_op), and the FlatMap kernels that
// expand table functions through the same MfpPlan (mzgpu_flat_map_new).
//
// Every row store of the operator is a segment: MZ_MFP_HDR header words (off[0..nb], the row range of
// each of its nb slices, written on the device) followed by the rows.  Row counts never come back to
// the host to launch the next kernel: grids are sized by host bounds and kernels read the lengths.
#include "common.cuh"

namespace {

constexpr int ET = 256;  // threads per block of every kernel here

// One row (words w, of which the MfpPlan reads the input words 0..2 and the extension words MZGPU_SRC_FN0.., and
// (time, diff)) through MfpPlan::evaluate (include/mzgpu.h), its map expressions evaluated lazily in
// SafeMfpPlan::evaluate_inner's order (mzgpu_mfp_new_map).  An output update at a time < upper (any time, if upper
// is MZGPU_FRONTIER_EMPTY) goes to the `ready` segment, any other to `held`; errors to `errs` (R32).  Each
// segment's count is header word 1, the error count *err_len.  Every lane of the warp calls it (`valid` false: no
// row); slots are reserved once per warp.  load(w) fills the row's words (NWW of them, zeroed) and returns
// its (time, diff).
template <int OW, int NWW, class Load>
__device__ __forceinline__ void mfp_eval_row(bool valid, Load load, const MfpDevPlan& pl, u64 upper, u64 until,
                                             u64* __restrict__ ready, u64* __restrict__ held,
                                             u64* __restrict__ errs, u64* __restrict__ err_len) {
  constexpr int ONW = OW / 8;
  u64 w[NWW] = {};
  u64 mv[MZGPU_MFP_MAX_MAPS];  // expression values
  u64 time = 0, diff = 0;
  // outputs: up to two updates (time, diff) and one error (code, payload)
  u32 n_upd = 0, e_code = 0;
  u64 t0 = 0, t1 = 0, e_pay = 0;
  if (valid) {
    const ulonglong2 td = load(w);
    time = td.x;
    diff = td.y;
    bool keep = mfp_filter_map(pl, w, mv, &e_code, &e_pay);
    u64 lower = time;
    for (u32 b = 0; b < pl.n_lower && keep; ++b) {
      const int q = pl.lower[b] & 7;
      MVal m = mfp_run(pl.plan.temporal_ops[q], pl.plan.n_temporal_ops[q], pl.plan.consts, pl.iv_us, w, mv);
      if (!m.err && (pl.lower[b] & 8)) {  // step_mz_timestamp
        if (m.v == ~0ull) m.err = MZGPU_MFP_ERR_MZ_TIMESTAMP_STEP_OVERFLOW;
        else m.v += 1;
      }
      if (m.err) {
        e_code = m.err;
        e_pay = m.pay;
        keep = false;
      } else if (m.v > lower) {
        lower = m.v;
      }
    }
    // valid(t) = t < until; until = MZGPU_FRONTIER_EMPTY (no until) makes every time valid
    if (keep && until != MZGPU_FRONTIER_EMPTY && lower >= until) keep = false;  // dropped before any upper bound
    bool has_up = false;
    u64 up = 0;
    for (u32 b = 0; b < pl.n_upper && keep; ++b) {
      if (has_up && up == lower) break;  // cannot be produced: later bounds are not evaluated
      const int q = pl.upper[b] & 7;
      MVal m = mfp_run(pl.plan.temporal_ops[q], pl.plan.n_temporal_ops[q], pl.plan.consts, pl.iv_us, w, mv);
      if (!m.err && (pl.upper[b] & 8)) {
        if (m.v == ~0ull) m.err = MZGPU_MFP_ERR_MZ_TIMESTAMP_STEP_OVERFLOW;
        else m.v += 1;
      }
      if (m.err) {
        e_code = m.err;
        e_pay = m.pay;
        keep = false;
      } else {
        up = has_up && up < m.v ? up : m.v;
        has_up = true;
        if (up < lower) up = lower;
      }
    }
    if (keep) {
      if (has_up && until != MZGPU_FRONTIER_EMPTY && up >= until) has_up = false;
      if (!(has_up && up == lower)) {
        t0 = lower;
        t1 = up;
        n_upd = has_up ? 2 : 1;
      }
    }
  }
  // route: ready (time < upper) or held
  const bool r0 = n_upd >= 1 && (upper == MZGPU_FRONTIER_EMPTY || t0 < upper);
  const bool r1 = n_upd >= 2 && (upper == MZGPU_FRONTIER_EMPTY || t1 < upper);
  const u32 c_ready = (u32)r0 + (u32)r1, c_held = n_upd - c_ready;
  const u64 p_ready = warp_reserve(c_ready, (unsigned long long*)(ready + 1));
  const u64 p_held = warp_reserve(c_held, (unsigned long long*)(held + 1));
  const u64 p_err = warp_reserve(e_code ? 1u : 0u, (unsigned long long*)err_len);
  u64 o[3] = {0, 0, 0};
  mfp_project<ONW>(pl, w, mv, o);
  u64 kr = p_ready, kh = p_held;
  for (u32 u = 0; u < n_upd; ++u) {
    const u64 t = u == 0 ? t0 : t1;
    const bool rd = u == 0 ? r0 : r1;
    u64* dst = (rd ? ready : held) + MZ_MFP_HDR + (rd ? kr++ : kh++) * ONW;
#pragma unroll
    for (int k = 0; k < ONW - 2; ++k) dst[k] = o[k];
    dst[ONW - 2] = t;
    dst[ONW - 1] = u == 0 ? diff : (u64)0 - diff;
  }
  if (e_code) {
    u64* dst = errs + p_err * 4;
    dst[0] = e_code;
    dst[1] = e_pay;
    dst[2] = time;
    dst[3] = diff;
  }
}

// k_mfp_eval<IW, OW>: every input row through mfp_eval_row.
template <int IW, int OW>
__global__ void __launch_bounds__(ET) k_mfp_eval(const u64* __restrict__ in, const DLen dn,
                                                  const __grid_constant__ MfpDevPlan pl, u64 upper, u64 until,
                                                  u64* __restrict__ ready, u64* __restrict__ held,
                                                  u64* __restrict__ errs, u64* __restrict__ err_len) {
  constexpr int INW = IW / 8;
  const u64 n = dlen_get(dn);
  const u64 stride = (u64)gridDim.x * ET;
  for (u64 base = (u64)blockIdx.x * ET; base < n; base += stride) {  // warp-uniform trip count
    const u64 i = base + threadIdx.x;
    auto load = [&](u64(&w)[3]) {
      const u64* r = in + i * INW;
      w[0] = r[0];
      w[1] = r[1];
      if (INW == 5) w[2] = r[2];
      return make_ulonglong2(r[INW - 2], r[INW - 1]);
    };
    mfp_eval_row<OW, 3>(i < n, load, pl, upper, until, ready, held, errs, err_len);
  }
}

// ------------------------------------------------------------------ FlatMap (mzgpu_flat_map_new)
typedef unsigned __int128 u128;
__device__ __forceinline__ u128 u128_of(const ulonglong2& v) { return ((u128)v.y << 64) | v.x; }
__device__ __forceinline__ ulonglong2 u128_split(u128 v) { return make_ulonglong2((u64)v, (u64)(v >> 64)); }

// range_step_inclusive(start, stop, step) has floor((stop - start) / step) + 1 values when the direction matches
// (its checked-add overflow stop never cuts a value <= stop short); up to 2^64
__device__ __forceinline__ u128 fm_series_count(i64 start, i64 stop, i64 step) {
  if (step > 0 && start <= stop) return (u128)(((u64)stop - (u64)start) / (u64)step) + 1;
  if (step < 0 && start >= stop) return (u128)(((u64)start - (u64)stop) / ((u64)0 - (u64)step)) + 1;
  return 0;
}

// One input row through the argument programs and the function (include/mzgpu.h, mzgpu_flat_map_new): its record,
// its function-row count, or an error (*e_code != 0).
__device__ __forceinline__ u128 fm_eval_func(const FlatMapDevPlan& pl, const u64* w, FmRec* rc, u32* e_code,
                                             u64* e_pay) {
  i64 a[3] = {0, 0, 0};
  for (u32 k = 0; k < pl.n_args; ++k) {
    const MVal m = mfp_run(pl.tf.ops[k], pl.tf.n_ops[k], pl.tf.consts, pl.iv_us, w, nullptr);
    if (m.err) {
      *e_code = m.err;
      *e_pay = m.pay;
      return 0;
    }
    a[k] = (i64)m.v;
  }
  const u32 kind = pl.tf.kind;
  rc->start = 0;
  rc->step = 0;
  rc->mult = 1;
  if (kind <= MZGPU_TF_GENERATE_SERIES_TIMESTAMP) {
    const i64 step = kind == MZGPU_TF_GENERATE_SERIES_TIMESTAMP ? pl.step_us : a[2];
    if (step == 0) {  // "step size cannot equal zero"
      *e_code = MZGPU_TF_ERR_INVALID_PARAMETER_VALUE;
      *e_pay = 0;
      return 0;
    }
    rc->start = a[0];
    rc->step = step;
    return fm_series_count(a[0], a[1], step);
  }
  const i64 n = a[0];
  if (kind == MZGPU_TF_REPEAT_ROW) {
    rc->mult = n;
    return n != 0 ? 1 : 0;
  }
  if (kind == MZGPU_TF_REPEAT_ROW_NON_NEGATIVE) {
    if (n < 0) {
      *e_code = MZGPU_TF_ERR_INVALID_PARAMETER_VALUE;
      *e_pay = (u64)n;
      return 0;
    }
    if (n == 0) return 0;
    if (!pl.tf.with_ordinality) {
      rc->mult = n;
      return 1;
    }
    rc->start = 1;  // n unit rows: the ordinal is column 0, 1 + j
    rc->step = 1;
    return (u128)n;
  }
  // MZGPU_TF_GUARD_SUBQUERY_SIZE
  if (n != 1) {
    *e_code = n > 1 ? MZGPU_TF_ERR_MULTIPLE_ROWS_FROM_SUBQUERY
                    : n < 0 ? MZGPU_TF_ERR_NEGATIVE_ROWS_FROM_SUBQUERY : MZGPU_TF_ERR_INTERNAL;
    *e_pay = 0;
  }
  return 0;
}

// inclusive block scan of one u128 per thread (ET threads); *tot gets the block's sum
__device__ __forceinline__ u128 fm_block_scan(u128 v, u128* s_warp, u128* tot) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u64 lo = __shfl_up_sync(0xffffffffu, (u64)v, d), hi = __shfl_up_sync(0xffffffffu, (u64)(v >> 64), d);
    if (lane >= d) v += ((u128)hi << 64) | lo;
  }
  if (lane == 31) s_warp[wid] = v;
  __syncthreads();
  u128 before = 0, all = 0;
  for (int k = 0; k < ET / 32; ++k) {
    if (k < wid) before += s_warp[k];
    all += s_warp[k];
  }
  __syncthreads();  // s_warp is reused by the next call
  *tot = all;
  return before + v;
}

// k_fm_count<IW>: every input row through fm_eval_func, and the inclusive 128-bit scan of the counts in one pass
// (tiles of MZ_FM_TILE rows in ticket order, each publishing its sum and then its inclusive prefix: a chained scan
// with decoupled look-back, whose predecessors have all started, so the look-back cannot deadlock).  State per
// tile: [flag, sum lo, sum hi, inclusive lo, inclusive hi]; flag 1 = sum published, 2 = inclusive published.  The
// last tile writes (total lo, total hi, n) to `total`.
template <int IW>
__global__ void __launch_bounds__(ET) k_fm_count(const u64* __restrict__ in, const DLen dn,
                                                  const __grid_constant__ FlatMapDevPlan pl, FmRec* __restrict__ rec,
                                                  ulonglong2* __restrict__ incl, u64* lb, u32* ticket, u64 n_tiles,
                                                  u64* __restrict__ total, u64* __restrict__ errs,
                                                  u64* __restrict__ err_len) {
  constexpr int INW = IW / 8, PER = MZ_FM_TILE / ET;
  __shared__ u32 s_tile;
  __shared__ u128 s_warp[ET / 32];
  __shared__ u128 s_prefix;
  const u64 n = dlen_get(dn);
  if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const u64 tile = s_tile;
  const u64 base = tile * MZ_FM_TILE;
  u128 mine[PER];
  u128 carry = 0;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const u64 i = base + (u64)k * ET + threadIdx.x;
    u128 c = 0;
    u32 e_code = 0;
    u64 e_pay = 0, time = 0, diff = 0;
    if (i < n) {
      const u64* r = in + i * INW;
      const u64 w[3] = {r[0], r[1], INW == 5 ? r[2] : 0};
      time = r[INW - 2];
      diff = r[INW - 1];
      FmRec rc;
      c = fm_eval_func(pl, w, &rc, &e_code, &e_pay);
      rec[i] = rc;
    }
    const u64 p_err = warp_reserve(e_code ? 1u : 0u, (unsigned long long*)err_len);
    if (e_code) {
      u64* dst = errs + p_err * 4;
      dst[0] = e_code;
      dst[1] = e_pay;
      dst[2] = time;
      dst[3] = diff;
    }
    u128 tot;
    mine[k] = carry + fm_block_scan(c, s_warp, &tot);
    carry += tot;
  }
  if (threadIdx.x == 0) {
    volatile u64* st = lb + tile * 5;
    u128 prefix = 0;
    if (tile > 0) {
      st[1] = (u64)carry;
      st[2] = (u64)(carry >> 64);
      __threadfence();
      st[0] = 1;
      for (u64 j = tile; j-- > 0;) {
        volatile u64* pj = lb + j * 5;
        u64 f;
        while ((f = pj[0]) == 0) {
        }
        __threadfence();
        if (f == 2) {
          prefix += ((u128)pj[4] << 64) | pj[3];
          break;
        }
        prefix += ((u128)pj[2] << 64) | pj[1];
      }
    }
    const u128 inc = prefix + carry;
    st[3] = (u64)inc;
    st[4] = (u64)(inc >> 64);
    __threadfence();
    st[0] = 2;
    s_prefix = prefix;
    if (tile == n_tiles - 1) {
      total[0] = (u64)inc;
      total[1] = (u64)(inc >> 64);
      total[2] = n;
    }
  }
  __syncthreads();
  const u128 prefix = s_prefix;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const u64 i = base + (u64)k * ET + threadIdx.x;
    if (i < n) incl[i] = u128_split(prefix + mine[k]);
  }
}

// the first row in [lo, hi) whose inclusive count exceeds ordinal o (hi if none)
__device__ __forceinline__ u64 fm_row_of(const ulonglong2* __restrict__ incl, u64 lo, u64 hi, u128 o) {
  while (lo < hi) {
    const u64 mid = lo + (hi - lo) / 2;
    if (u128_of(incl[mid]) > o) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

// k_fm_expand<IW, OW>: function rows [g, g + page) of the activation, load-balanced: each tile of ET ordinals finds
// its first and last source rows by binary search over the scan, and each ordinal its row within them.  Ordinal o
// of row i is function row j = o - (inclusive count of row i - 1's) of that row: the extension columns
// (start + j * step, then the ordinal j + 1) after the input words, at the input's time with diff
// mult * diff, through mfp_eval_row.
template <int IW, int OW>
__global__ void __launch_bounds__(ET) k_fm_expand(const u64* __restrict__ in, const FmRec* __restrict__ rec,
                                                   const ulonglong2* __restrict__ incl, u64 n, u64 g_lo, u64 g_hi,
                                                   u64 page, const __grid_constant__ FlatMapDevPlan pl, u64 upper,
                                                   u64 until, u64* __restrict__ ready, u64* __restrict__ held,
                                                   u64* __restrict__ errs, u64* __restrict__ err_len) {
  constexpr int INW = IW / 8;
  __shared__ u64 s_r[2];
  const u128 g = ((u128)g_hi << 64) | g_lo;
  const u64 stride = (u64)gridDim.x * ET;
  for (u64 tb = (u64)blockIdx.x * ET; tb < page; tb += stride) {  // block-uniform trip count
    const u64 last = min(tb + ET, page) - 1;
    __syncthreads();
    if (threadIdx.x == 0) s_r[0] = fm_row_of(incl, 0, n, g + tb);
    if (threadIdx.x == 32) s_r[1] = fm_row_of(incl, 0, n, g + last);
    __syncthreads();
    const u64 t = tb + threadIdx.x;
    const bool valid = t < page;
    const u128 o = g + t;
    const u64 i = valid ? fm_row_of(incl, s_r[0], s_r[1] + 1, o) : 0;
    auto load = [&](u64(&w)[MZGPU_SRC_FN0 + 2]) {
      const u64* r = in + i * INW;
      w[0] = r[0];
      w[1] = r[1];
      if (INW == 5) w[2] = r[2];
      const u128 before = i ? u128_of(incl[i - 1]) : 0;
      const u64 j = (u64)(o - before);
      const FmRec rc = rec[i];
      w[MZGPU_SRC_FN0] = (u64)rc.start + j * (u64)rc.step;
      w[MZGPU_SRC_FN0 + 1] = j + 1;
      return make_ulonglong2(r[INW - 2], (u64)rc.mult * r[INW - 1]);
    };
    mfp_eval_row<OW, MZGPU_SRC_FN0 + 2>(valid, load, pl.mfp, upper, until, ready, held, errs, err_len);
  }
}

// the least input time among rows with function rows at ordinals >= g
template <int IW>
__global__ void __launch_bounds__(ET) k_fm_min_time(const u64* __restrict__ in, const ulonglong2* __restrict__ incl,
                                                     u64 n, u64 g_lo, u64 g_hi, u64* __restrict__ m) {
  constexpr int INW = IW / 8;
  const u128 g = ((u128)g_hi << 64) | g_lo;
  u64 best = ~0ull;
  for (u64 i = (u64)blockIdx.x * ET + threadIdx.x; i < n; i += (u64)gridDim.x * ET) {
    const u128 hi = u128_of(incl[i]), lo = i ? u128_of(incl[i - 1]) : 0;
    if (hi > g && hi > lo) best = min(best, in[i * INW + INW - 2]);
  }
  if (best != ~0ull) atomicMin((unsigned long long*)m, (unsigned long long)best);
}

// the slot of time t among bounds b[0..nb): (# bounds <= t) - 1, at least 0
__device__ __forceinline__ u32 mfp_slot(const MfpBounds& b, u64 t) {
  u32 lo = 0, hi = b.nb;
  while (lo < hi) {
    const u32 mid = (lo + hi) >> 1;
    if (b.v[mid] <= t) lo = mid + 1;
    else hi = mid;
  }
  return lo ? lo - 1 : 0;
}

// pass 1 of a partition: per-slot histogram of the source slices' rows
template <int NW>
__global__ void __launch_bounds__(ET) k_mfp_count(const MfpSlices s, const __grid_constant__ MfpBounds b,
                                                   u64* __restrict__ hist, u64* __restrict__ touched) {
  __shared__ u32 h[MZ_MFP_MAX_SLOTS];
  __shared__ unsigned long long seen_blk;
  for (u32 j = threadIdx.x; j < b.nb; j += ET) h[j] = 0;
  if (threadIdx.x == 0) seen_blk = 0;
  __syncthreads();
  const u64 gtid = (u64)blockIdx.x * ET + threadIdx.x, stride = (u64)gridDim.x * ET;
  u64 seen = 0;
  for (u32 k = 0; k < s.n; ++k) {
    const u64* seg = s.base[k];
    const u64 lo = seg[s.idx[k]], hi = seg[s.idx[k] + 1];
    const u64* rows = seg + MZ_MFP_HDR;
    for (u64 i = lo + gtid; i < hi; i += stride) {
      atomicAdd(&h[mfp_slot(b, rows[i * NW + NW - 2])], 1u);
      ++seen;
    }
  }
  __syncthreads();
  if (seen) atomicAdd(&seen_blk, (unsigned long long)seen);
  __syncthreads();
  for (u32 j = threadIdx.x; j < b.nb; j += ET)
    if (h[j]) atomicAdd((unsigned long long*)&hist[j], (unsigned long long)h[j]);
  if (threadIdx.x == 0 && seen_blk) atomicAdd((unsigned long long*)touched, seen_blk);  // one global add per block
}

// pass 2: scatter every row to its slot of the destination segment (order within a slot is arbitrary:
// every release is consolidated); block 0 writes the segment header and the total
template <int NW>
__global__ void __launch_bounds__(ET) k_mfp_scatter(const MfpSlices s, const __grid_constant__ MfpBounds b,
                                                     const u64* __restrict__ hist, u64* __restrict__ cursor,
                                                     u64* __restrict__ dst, u64* __restrict__ total,
                                                     u64* __restrict__ touched) {
  __shared__ u64 off[MZ_MFP_MAX_SLOTS + 1];
  __shared__ unsigned long long moved_blk;
  if (threadIdx.x == 0) {
    moved_blk = 0;
    u64 a = 0;
    for (u32 j = 0; j < b.nb; ++j) {
      off[j] = a;
      a += hist[j];
    }
    off[b.nb] = a;
    if (blockIdx.x == 0) {
      for (u32 j = 0; j <= b.nb; ++j) dst[j] = off[j];
      if (total) *total = a;
    }
  }
  __syncthreads();
  const u64 gtid = (u64)blockIdx.x * ET + threadIdx.x, stride = (u64)gridDim.x * ET;
  u64 moved = 0;
  u64* out = dst + MZ_MFP_HDR;
  for (u32 k = 0; k < s.n; ++k) {
    const u64* seg = s.base[k];
    const u64 lo = seg[s.idx[k]], hi = seg[s.idx[k] + 1];
    const u64* rows = seg + MZ_MFP_HDR;
    for (u64 i = lo + gtid; i < hi; i += stride) {
      const u64* r = rows + i * NW;
      const u32 j = mfp_slot(b, r[NW - 2]);
      // one cursor reservation per warp and slot (a split has 2 slots, a gather 1: per-row atomics on one
      // address would serialise)
      const unsigned act = __activemask();
      const unsigned peers = __match_any_sync(act, j);
      const int leader = __ffs(peers) - 1;
      const unsigned lane = threadIdx.x & 31;
      unsigned long long base = 0;
      if ((int)lane == leader) base = atomicAdd((unsigned long long*)&cursor[j], (unsigned long long)__popc(peers));
      base = __shfl_sync(peers, base, leader);
      const u64 p = off[j] + base + __popc(peers & ((1u << lane) - 1));
#pragma unroll
      for (int q = 0; q < NW; ++q) out[p * NW + q] = r[q];
      ++moved;
    }
  }
  if (moved) atomicAdd(&moved_blk, (unsigned long long)moved);
  __syncthreads();
  if (threadIdx.x == 0 && moved_blk) atomicAdd((unsigned long long*)touched, moved_blk);
}

// the least time of the source slices' rows (atomicMin into *m, which starts at u64::MAX)
template <int NW>
__global__ void __launch_bounds__(ET) k_mfp_min_time(const MfpSlices s, u64* __restrict__ m) {
  const u64 gtid = (u64)blockIdx.x * ET + threadIdx.x, stride = (u64)gridDim.x * ET;
  u64 best = ~0ull;
  for (u32 k = 0; k < s.n; ++k) {
    const u64* seg = s.base[k];
    const u64 lo = seg[s.idx[k]], hi = seg[s.idx[k] + 1];
    const u64* rows = seg + MZ_MFP_HDR;
    for (u64 i = lo + gtid; i < hi; i += stride) best = min(best, rows[i * NW + NW - 2]);
  }
  if (best != ~0ull) atomicMin((unsigned long long*)m, (unsigned long long)best);
}

static unsigned mfp_grid(mzgpu_ctx* ctx, u64 n_ub) {
  u64 g = (n_ub + ET - 1) / ET;
  const u64 maxg = (u64)ctx->num_sms * 8;
  if (g > maxg) g = maxg;
  return g == 0 ? 1u : (unsigned)g;
}

}  // namespace

int32_t mz_mfp_eval(mzgpu_ctx* ctx, const MfpDevPlan& pl, const u64* d_rows, DLen n, u64 n_ub, u64 upper, u64 until,
                    u64* ready, u64* held, u64* errs, u64* err_len) {
  const int iw = (int)pl.plan.in_row_bytes, ow = (int)pl.plan.out_row_bytes;
  const unsigned grid = mfp_grid(ctx, n_ub);
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * (u64)(iw + 2 * ow) : 0);
  if (iw == 32 && ow == 32) MZ_LAUNCH(ctx, (k_mfp_eval<32, 32>), grid, ET, 0, d_rows, n, pl, upper, until, ready, held, errs, err_len);
  else if (iw == 32) MZ_LAUNCH(ctx, (k_mfp_eval<32, 40>), grid, ET, 0, d_rows, n, pl, upper, until, ready, held, errs, err_len);
  else if (ow == 32) MZ_LAUNCH(ctx, (k_mfp_eval<40, 32>), grid, ET, 0, d_rows, n, pl, upper, until, ready, held, errs, err_len);
  else MZ_LAUNCH(ctx, (k_mfp_eval<40, 40>), grid, ET, 0, d_rows, n, pl, upper, until, ready, held, errs, err_len);
  return MZGPU_OK;
}

int32_t mz_mfp_partition(mzgpu_ctx* ctx, int rb, const MfpSlices* chunks, u32 n_chunks, u64 rows_ub,
                         const MfpBounds& b, u64* hist, u64* cursor, u64* dst, u64* total, u64* touched) {
  const unsigned grid = mfp_grid(ctx, rows_ub);
  MZ_CUDA(ctx, cudaMemsetAsync(hist, 0, 2 * MZ_MFP_MAX_SLOTS * sizeof(u64), ctx->stream));  // hist + cursor
  for (u32 c = 0; c < n_chunks; ++c) {
    if (rb == 32) MZ_LAUNCH(ctx, k_mfp_count<4>, grid, ET, 0, chunks[c], b, hist, touched);
    else MZ_LAUNCH(ctx, k_mfp_count<5>, grid, ET, 0, chunks[c], b, hist, touched);
  }
  for (u32 c = 0; c < n_chunks; ++c) {
    MZ_BYTES(ctx, 0);
    if (rb == 32) MZ_LAUNCH(ctx, k_mfp_scatter<4>, grid, ET, 0, chunks[c], b, hist, cursor, dst, total, touched);
    else MZ_LAUNCH(ctx, k_mfp_scatter<5>, grid, ET, 0, chunks[c], b, hist, cursor, dst, total, touched);
  }
  return MZGPU_OK;
}

int32_t mz_mfp_min_time(mzgpu_ctx* ctx, int rb, const MfpSlices* chunks, u32 n_chunks, u64 rows_ub, u64* d_min) {
  const unsigned grid = mfp_grid(ctx, rows_ub);
  MZ_CUDA(ctx, cudaMemsetAsync(d_min, 0xff, sizeof(u64), ctx->stream));
  for (u32 c = 0; c < n_chunks; ++c) {
    if (rb == 32) MZ_LAUNCH(ctx, k_mfp_min_time<4>, grid, ET, 0, chunks[c], d_min);
    else MZ_LAUNCH(ctx, k_mfp_min_time<5>, grid, ET, 0, chunks[c], d_min);
  }
  return MZGPU_OK;
}

int32_t mz_fm_count(mzgpu_ctx* ctx, const FlatMapDevPlan& pl, const u64* d_rows, DLen n, u64 n_ub, FmRec* rec,
                    ulonglong2* incl, u64* lb_state, u64* d_total, u64* errs, u64* err_len) {
  const u64 n_tiles = n_ub == 0 ? 1 : (n_ub + MZ_FM_TILE - 1) / MZ_FM_TILE;
  u32* ticket = (u32*)(lb_state + n_tiles * 5);
  MZ_CUDA(ctx, cudaMemsetAsync(lb_state, 0, (n_tiles * 5 + 1) * sizeof(u64), ctx->stream));
  MZ_BYTES(ctx, 0);
  if (pl.mfp.plan.in_row_bytes == 32)
    MZ_LAUNCH(ctx, k_fm_count<32>, (unsigned)n_tiles, ET, 0, d_rows, n, pl, rec, incl, lb_state, ticket, n_tiles,
              d_total, errs, err_len);
  else
    MZ_LAUNCH(ctx, k_fm_count<40>, (unsigned)n_tiles, ET, 0, d_rows, n, pl, rec, incl, lb_state, ticket, n_tiles,
              d_total, errs, err_len);
  return MZGPU_OK;
}

int32_t mz_fm_expand(mzgpu_ctx* ctx, const FlatMapDevPlan& pl, const u64* d_rows, const FmRec* rec,
                     const ulonglong2* incl, u64 n, unsigned __int128 g, u64 page, u64 upper, u64 until, u64* ready,
                     u64* held, u64* errs, u64* err_len) {
  const int iw = (int)pl.mfp.plan.in_row_bytes, ow = (int)pl.mfp.plan.out_row_bytes;
  const unsigned grid = mfp_grid(ctx, page);
  const u64 g_lo = (u64)g, g_hi = (u64)(g >> 64);
  MZ_BYTES(ctx, page * (u64)(2 * ow));
  if (iw == 32 && ow == 32)
    MZ_LAUNCH(ctx, (k_fm_expand<32, 32>), grid, ET, 0, d_rows, rec, incl, n, g_lo, g_hi, page, pl, upper, until,
              ready, held, errs, err_len);
  else if (iw == 32)
    MZ_LAUNCH(ctx, (k_fm_expand<32, 40>), grid, ET, 0, d_rows, rec, incl, n, g_lo, g_hi, page, pl, upper, until,
              ready, held, errs, err_len);
  else if (ow == 32)
    MZ_LAUNCH(ctx, (k_fm_expand<40, 32>), grid, ET, 0, d_rows, rec, incl, n, g_lo, g_hi, page, pl, upper, until,
              ready, held, errs, err_len);
  else
    MZ_LAUNCH(ctx, (k_fm_expand<40, 40>), grid, ET, 0, d_rows, rec, incl, n, g_lo, g_hi, page, pl, upper, until,
              ready, held, errs, err_len);
  return MZGPU_OK;
}

int32_t mz_fm_min_time(mzgpu_ctx* ctx, int iw, const u64* d_rows, const ulonglong2* incl, u64 n,
                       unsigned __int128 g, u64* d_min) {
  const unsigned grid = mfp_grid(ctx, n);
  const u64 g_lo = (u64)g, g_hi = (u64)(g >> 64);
  if (iw == 32) MZ_LAUNCH(ctx, k_fm_min_time<32>, grid, ET, 0, d_rows, incl, n, g_lo, g_hi, d_min);
  else MZ_LAUNCH(ctx, k_fm_min_time<40>, grid, ET, 0, d_rows, incl, n, g_lo, g_hi, d_min);
  return MZGPU_OK;
}
