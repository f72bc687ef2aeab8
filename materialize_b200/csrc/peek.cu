// peek.cu — index peeks (mzgpu_peek_many): the gather of a trace's pairs at a timestamp, the MfpPlan over each
// accumulated pair, and the ORDER BY / LIMIT / OFFSET finishing.  The consolidations between the phases are the
// generic ones (consolidate_dev in host.cu); literal lookups run through the half-join probe.
#include "common.cuh"

namespace {

// Full scans: every row of every batch of the trace (a batch still being built through its device header) with
// time <= as_of becomes the R40 row (slot, key, val, as_of, diff).  Grid y = the job; rows are appended with one
// warp-aggregated reservation per warp and step (the loop bound is warp-uniform, so every lane reaches it).
__global__ void __launch_bounds__(256) k_peek_scan(const __grid_constant__ TraceView tv,
                                                   const __grid_constant__ PeekScanJobs jobs, u64* __restrict__ out,
                                                   u64 cap, unsigned long long* __restrict__ len) {
  const u32 j = blockIdx.y;
  const u64 slot = jobs.slot[j], as_of = jobs.as_of[j];
  const u32 lane = threadIdx.x & 31;
  const u64 stride = (u64)gridDim.x * 256;
  for (u32 b = 0; b < tv.n_batches; ++b) {
    const BatchView& bv = tv.b[b];
    const u64 n = bv_n(bv);
    for (u64 base = (u64)blockIdx.x * 256 + (threadIdx.x & ~31u); base < n; base += stride) {
      const u64 i = base + lane;
      u64 r[4] = {0, 0, 0, 0};
      bool keep = false;
      if (i < n) {
        const ulonglong2* p = reinterpret_cast<const ulonglong2*>(bv.rows + i * 4);
        const ulonglong2 a = p[0], c = p[1];
        r[0] = a.x;
        r[1] = a.y;
        r[2] = c.x;
        r[3] = c.y;
        keep = r[2] <= as_of;
      }
      const u64 pos = warp_reserve(keep ? 1u : 0u, len);
      if (keep && pos < cap) {
        u64* o = out + pos * 5;
        o[0] = slot;
        o[1] = r[0];
        o[2] = r[1];
        o[3] = as_of;
        o[4] = r[3];
      }
    }
  }
}

// Literal keys -> the probe's stream rows (key, slot, as_of, +1).
__global__ void __launch_bounds__(256) k_peek_lits(const u64* __restrict__ keys, const __grid_constant__ PeekLitSegs segs,
                                                   u64* __restrict__ rows) {
  const u64 n = segs.start[segs.n];
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) {
    u32 s = 0;
    while (s + 1 < segs.n && segs.start[s + 1] <= i) ++s;
    u64* o = rows + i * 4;
    o[0] = keys[i];
    o[1] = segs.slot[s];
    o[2] = segs.as_of[s];
    o[3] = 1;
  }
}

// Consolidated stream rows: a duplicate literal counts once (the reference's forward-only seek).
__global__ void __launch_bounds__(256) k_peek_unit(u64* __restrict__ rows, const DLen dn) {
  const u64 n = dlen_get(dn);
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) rows[i * 4 + 3] = 1;
}

__device__ __forceinline__ void peek_order(const PeekFin& f, const u64* o, u64* e) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    u64 v = 0;
    if ((u32)j < f.n_order) {
      v = field_get(f.f[j], o[0], o[1], o[2]);
      const u32 bits = f.f[j].bits;
      if (f.sign_extend[j] && bits < 64 && ((v >> (bits - 1)) & 1)) v |= ~0ull << bits;
      v ^= f.xm[j];
    }
    e[j] = v;
  }
}

// One pair per thread, for every request of its slot: the request's MfpPlan over (key, val).  An error, or a kept pair
// with a negative count, is a failure (the least row index per request wins: a request's pairs are one slot's rows,
// in (key, val) order); a kept pair becomes a finishing row led by the request.  Error-trace slots only record their
// first row.  The requests are walked over the warp's union of bit sets, so every lane reaches each reservation.
__global__ void __launch_bounds__(256) k_peek_eval(const u64* __restrict__ pairs, const DLen dn,
                                                   const __grid_constant__ PeekReqs rq, u64* __restrict__ fin,
                                                   u64 fin_cap, unsigned long long* __restrict__ fin_len,
                                                   unsigned long long* __restrict__ fail) {
  const u64 n = dlen_get(dn);
  const u32 lane = threadIdx.x & 31;
  const u64 stride = (u64)gridDim.x * 256;
  for (u64 base = (u64)blockIdx.x * 256 + (threadIdx.x & ~31u); base < n; base += stride) {
    const u64 i = base + lane;
    const u64* r = pairs + i * 5;
    u64 mine = 0;
    if (i < n) {
      const u64 slot = r[0];
      if (slot >= rq.err_base)
        atomicMin(fail + slot, (unsigned long long)i);
      else
        mine = rq.reqs[slot];
    }
    const u64 all = ((u64)__reduce_or_sync(0xffffffffu, (u32)(mine >> 32)) << 32) |
                    __reduce_or_sync(0xffffffffu, (u32)mine);
    for (u64 left = all; left != 0; left &= left - 1) {
      const u32 q = (u32)__ffsll((long long)left) - 1;
      bool emit = false;
      u64 row[9];
      if ((mine >> q) & 1) {
        const PeekDevPlan& pl = *rq.pl[q];
        const u64 w[3] = {r[1], r[2], 0};
        u64 mv[MZGPU_MFP_MAX_MAPS];
        u32 e_code = 0;
        u64 e_pay = 0;
        const bool keep = mfp_filter_map(pl.mfp, w, mv, &e_code, &e_pay);
        const i64 c = (i64)r[4];
        if (e_code != 0 || (keep && c < 0)) {
          atomicMin(fail + q, (unsigned long long)i);
        } else if (keep) {
          u64 o[3];
          mfp_project<5>(pl.mfp, w, mv, o);
          row[0] = q;
          peek_order(pl.fin, o, row + 1);
          row[4] = o[0];
          row[5] = o[1];
          row[6] = o[2];
          row[7] = (u64)c;
          row[8] = 0;
          emit = true;
        }
      }
      const u64 pos = warp_reserve(emit ? 1u : 0u, fin_len);
      if (emit && pos < fin_cap) {
        u64* o = fin + pos * 9;
#pragma unroll
        for (int w = 0; w < 9; ++w) o[w] = row[w];
      }
    }
  }
}

// exclusive block-wide prefix of v (256 threads); *total gets the sum
__device__ __forceinline__ u64 block_excl(u64 v, u64* sh, u64* total) {
  const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  u64 s = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u64 t = __shfl_up_sync(0xffffffffu, s, d);
    if (lane >= d) s += t;
  }
  if (lane == 31) sh[wid] = s;
  __syncthreads();
  u64 before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    if ((u32)w < wid) before += sh[w];
    all += sh[w];
  }
  __syncthreads();
  *total = all;
  return before + s - v;
}

__device__ __forceinline__ u64 lower_bound_slot(const u64* fin, u64 n, u64 slot) {
  u64 lo = 0, hi = n;
  while (lo < hi) {
    const u64 mid = (lo + hi) / 2;
    if (fin[mid * 9] < slot)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// Block = request.  A failed request gets its detail (the first row of its error-trace slot first, then its first
// failing pair, re-evaluated for its error); otherwise its finishing rows (sorted) are cut to units [offset, end) and
// projected into the staging rows at byte offset lo * 40, where lo is the request's first finishing row.
__global__ void __launch_bounds__(256) k_peek_finish(const __grid_constant__ PeekReqs rq, const u64* __restrict__ pairs,
                                                     const unsigned long long* __restrict__ fail,
                                                     const u64* __restrict__ fin, const DLen dn,
                                                     u64* __restrict__ stage, PeekDevResult* __restrict__ res) {
  __shared__ u64 sh[8];
  const u32 q = blockIdx.x;
  if (rq.pl[q] == nullptr) return;
  const PeekDevPlan& pl = *rq.pl[q];
  PeekDevResult* R = res + q;
  const int es = rq.err_slot[q];
  const u64 ef = es >= 0 ? fail[es] : ~0ull;
  const u64 f = fail[q];
  if (ef != ~0ull || f != ~0ull) {
    if (threadIdx.x == 0) {
      const u64* r = pairs + (ef != ~0ull ? ef : f) * 5;
      R->n_rows = 0;
      R->lo = 0;
      if (ef != ~0ull) {
        R->kind = (i64)r[4] > 0 ? MZGPU_PEEK_ERR_ERRS_ROW : MZGPU_PEEK_ERR_ERRS_RETRACTION;
        R->d[0] = r[1];
        R->d[1] = r[2];
        R->d[2] = (i64)r[4] > 0 ? 0 : r[4];
        R->d[3] = 0;
      } else {
        const u64 w[3] = {r[1], r[2], 0};
        u64 mv[MZGPU_MFP_MAX_MAPS];
        u32 e_code = 0;
        u64 e_pay = 0;
        mfp_filter_map(pl.mfp, w, mv, &e_code, &e_pay);
        if (e_code != 0) {
          R->kind = MZGPU_PEEK_ERR_MFP;
          R->d[0] = e_code;
          R->d[1] = e_pay;
          R->d[2] = r[1];
          R->d[3] = r[2];
        } else {
          R->kind = MZGPU_PEEK_ERR_RETRACTION;
          R->d[0] = r[1];
          R->d[1] = r[2];
          R->d[2] = r[4];
          R->d[3] = 0;
        }
      }
    }
    return;
  }
  const u64 n = dlen_get(dn);
  const u64 lo = lower_bound_slot(fin, n, q), hi = lower_bound_slot(fin, n, (u64)q + 1);
  const PeekFin& F = pl.fin;
  const u32 ow = F.out_words;
  const u64 as_of = rq.as_of[q];
  u64* dst = stage + lo * 5;
  u64 units = 0, written = 0;
  for (u64 base = lo; base < hi && units < F.end; base += 256) {
    const u64 i = base + threadIdx.x;
    const u64* r = fin + i * 9;
    const u64 c = i < hi ? r[7] : 0;
    u64 csum;
    const u64 s = units + block_excl(c, sh, &csum);
    const u64 e = s + c;  // units [s, e) of this row
    const u64 a = s > F.offset ? s : F.offset, b = e < F.end ? e : F.end;
    const u64 kept = b > a ? b - a : 0;
    u64 ksum;
    const u64 at = written + block_excl(kept ? 1 : 0, sh, &ksum);
    if (kept) {
      const u64 o[3] = {r[4], r[5], r[6]};
      u64* d = dst + at * (ow + 2);
      for (u32 w = 0; w < ow; ++w) {
        u64 v = o[w];
        if (!F.identity) {
          v = 0;
          for (u32 x = 0; x < F.n_project[w]; ++x) {
            const mzgpu_field& fd = F.project[w][x];
            v |= field_get(fd, o[0], o[1], o[2]) << fd.dst_shift;
          }
        }
        d[w] = v;
      }
      d[ow] = as_of;
      d[ow + 1] = kept;
    }
    units += csum;
    written += ksum;
  }
  if (threadIdx.x == 0) {
    R->kind = 0;
    R->n_rows = written;
    R->lo = lo;
    R->d[0] = R->d[1] = R->d[2] = R->d[3] = 0;
  }
}

unsigned peek_grid(mzgpu_ctx* ctx, u64 n_ub) {
  u64 g = (n_ub + 255) / 256;
  const u64 maxg = (u64)ctx->num_sms * 8;
  if (g > maxg) g = maxg;
  return g == 0 ? 1u : (unsigned)g;
}

}  // namespace

int32_t mz_peek_scan(mzgpu_ctx* ctx, const TraceView& tv, const PeekScanJobs& jobs, u64* d_out, u64 cap, u64* d_len) {
  if (jobs.n == 0 || tv.n_batches == 0) return MZGPU_OK;
  MZ_BYTES(ctx, cap / jobs.n * 32);
  // the grid's x extent shares one wave of blocks among the jobs
  const unsigned gx = peek_grid(ctx, cap / jobs.n) / jobs.n;
  const dim3 grid(gx > 0 ? gx : 1u, jobs.n);
  MZ_LAUNCH(ctx, k_peek_scan, grid, 256, 0, tv, jobs, d_out, cap, (unsigned long long*)d_len);
  return MZGPU_OK;
}

int32_t mz_peek_lits(mzgpu_ctx* ctx, const u64* d_keys, const PeekLitSegs& segs, u64* d_rows) {
  const u64 n = segs.start[segs.n];
  if (n == 0) return MZGPU_OK;
  MZ_BYTES(ctx, n * 40);
  MZ_LAUNCH(ctx, k_peek_lits, peek_grid(ctx, n), 256, 0, d_keys, segs, d_rows);
  return MZGPU_OK;
}

int32_t mz_peek_unit(mzgpu_ctx* ctx, u64* d_rows, DLen n, u64 n_ub) {
  if (n_ub == 0) return MZGPU_OK;
  MZ_BYTES(ctx, n_ub * 8);
  MZ_LAUNCH(ctx, k_peek_unit, peek_grid(ctx, n_ub), 256, 0, d_rows, n);
  return MZGPU_OK;
}

int32_t mz_peek_eval(mzgpu_ctx* ctx, const u64* d_pairs, DLen n, u64 n_ub, u64 fin_cap, const PeekReqs& rq, u64* d_fin,
                     u64* d_fin_len, u64* d_fail) {
  if (n_ub == 0) return MZGPU_OK;
  MZ_BYTES(ctx, n_ub * (40 + 72));
  MZ_LAUNCH(ctx, k_peek_eval, peek_grid(ctx, n_ub), 256, 0, d_pairs, n, rq, d_fin, fin_cap, (unsigned long long*)d_fin_len,
            (unsigned long long*)d_fail);
  return MZGPU_OK;
}

int32_t mz_peek_finish(mzgpu_ctx* ctx, const PeekReqs& rq, const u64* d_pairs, const u64* d_fail, const u64* d_fin,
                       DLen n_fin, u64* d_stage, PeekDevResult* d_res) {
  MZ_BYTES(ctx, 0);
  MZ_LAUNCH(ctx, k_peek_finish, rq.k, 256, 0, rq, d_pairs, (const unsigned long long*)d_fail, d_fin, n_fin, d_stage,
            d_res);
  return MZGPU_OK;
}
