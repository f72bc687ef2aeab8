// merge.cu — merge-path 2-way merge of sorted, consolidated update arrays
// (SURVEY.md a3, a7) and the seal-time extract (a4).
//
// Reference:
//   InternalMerge::merge_from      src/timely-util/src/columnation.rs:579-634
//   Merger::merge (chain merge)    src/timely-util/src/columnar/batcher.rs:635-753
//   Batch::Merger for OrdValBatch  differential-dataflow 0.23.0 (external), semantics
//                                  SURVEY.md A4: union, time.advance_by(since),
//                                  re-consolidate, drop empty vals/keys
//   InternalMerge::extract         src/timely-util/src/columnation.rs:636-655
//
// The CPU path walks two cursors row by row.  Here a partition kernel cuts the
// merge into equal-sized output tiles with one binary search per tile (merge
// path), each CTA stages its two input ranges in shared memory, every thread
// merges a fixed number of outputs, and the generic segmented-sum sweep
// (consolidate.cu) folds equal (key, val, time) neighbours afterwards.
// advance_by(since) = max(time, since) is monotone for totally ordered times
// (src/repr/src/timestamp.rs:486-495), so it can be applied on the fly without
// disturbing the sort order.
#include "common.cuh"

namespace {

constexpr int MT = 256;  // threads per merge CTA

template <int RB>
struct MergeCfg {
  static constexpr int VT = RB <= 40 ? 4 : 2;  // outputs per thread
  static constexpr int TILE = MT * VT;
};

template <int NK, int TW>
__device__ __forceinline__ bool keys_less(const u64* a, const u64* b, u64 since) {
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    u64 x = a[k], y = b[k];
    if (k == TW) {
      x = x < since ? since : x;
      y = y < since ? since : y;
    }
    if (x != y) return x < y;
  }
  return false;
}

// a_split[t] = number of A rows among the first min(t*TILE, na+nb) outputs
// (ties take A first: A is the older batch).
template <int RB>
__global__ void __launch_bounds__(256) k_merge_partition(const u64* __restrict__ A, u64 na,
                                                         const u64* __restrict__ B, u64 nb, u64 since,
                                                         u64 n_tiles, u64* __restrict__ a_split) {
  constexpr int NW = RowT<RB>::NW, NK = RowT<RB>::NK, TW = RowT<RB>::TW;
  constexpr u64 TILE = MergeCfg<RB>::TILE;
  u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (t > n_tiles) return;
  u64 diag = t * TILE;
  if (diag > na + nb) diag = na + nb;
  u64 lo = diag > nb ? diag - nb : 0;
  u64 hi = diag < na ? diag : na;
  while (lo < hi) {
    u64 mid = (lo + hi) >> 1;
    u64 b = diag - mid;  // >= 1
    if (!keys_less<NK, TW>(B + (b - 1) * NW, A + mid * NW, since))
      lo = mid + 1;
    else
      hi = mid;
  }
  a_split[t] = lo;
}

template <int RB>
__global__ void __launch_bounds__(MT) k_merge_tiles(const u64* __restrict__ A, u64 na,
                                                    const u64* __restrict__ B, u64 nb, u64 since,
                                                    const u64* __restrict__ a_split,
                                                    u64* __restrict__ out) {
  constexpr int NW = RowT<RB>::NW, NK = RowT<RB>::NK, TW = RowT<RB>::TW;
  constexpr int VT = MergeCfg<RB>::VT;
  constexpr u32 TILE = MergeCfg<RB>::TILE;
  // rows wider than RACC do not fit a tile in shared memory: only their sort keys are staged
  // there (SW words per row), and the output copies each row from global memory
  constexpr bool KEYS_ONLY = NW > 10;
  constexpr int SW = KEYS_ONLY ? NK : NW;
  __shared__ __align__(16) u64 sm[TILE * SW];
  const u64 t = blockIdx.x;
  const u64 diag0 = t * TILE;
  u64 diag1 = diag0 + TILE;
  if (diag1 > na + nb) diag1 = na + nb;
  const u64 a0 = a_split[t], a1 = a_split[t + 1];
  const u64 b0 = diag0 - a0, b1 = diag1 - a1;
  const u32 ca = (u32)(a1 - a0), cb = (u32)(b1 - b0);
  // stage both ranges; times advanced on the way in
  for (u32 i = threadIdx.x; i < ca + cb; i += MT) {
    u64 r[SW];
    if (KEYS_ONLY) {
      const u64* g = i < ca ? A + (a0 + i) * NW : B + (b0 + (i - ca)) * NW;
#pragma unroll
      for (int w = 0; w < SW; ++w) r[w] = g[w];
    } else if (i < ca) {
      load_row<SW>(A, a0 + i, r);
    } else {
      load_row<SW>(B, b0 + (i - ca), r);
    }
    if (TW >= 0) r[TW >= 0 ? TW : 0] = r[TW >= 0 ? TW : 0] < since ? since : r[TW >= 0 ? TW : 0];
#pragma unroll
    for (int w = 0; w < SW; ++w) sm[(u64)i * SW + w] = r[w];
  }
  __syncthreads();
  const u64* sa = sm;
  const u64* sb = sm + (u64)ca * SW;
  // per-thread merge path inside the tile
  u32 d = threadIdx.x * VT;
  const u32 total = ca + cb;
  if (d > total) d = total;
  u32 lo = d > cb ? d - cb : 0, hi = d < ca ? d : ca;
  while (lo < hi) {
    u32 mid = (lo + hi) >> 1;
    u32 b = d - mid;
    if (!keys_less<NK, -1>(sb + (u64)(b - 1) * SW, sa + (u64)mid * SW, 0))
      lo = mid + 1;
    else
      hi = mid;
  }
  u32 ia = lo, ib = d - lo;
#pragma unroll
  for (int k = 0; k < VT; ++k) {
    u32 o = d + k;
    if (o >= total) break;
    bool take_a;
    if (ia >= ca)
      take_a = false;
    else if (ib >= cb)
      take_a = true;
    else
      take_a = !keys_less<NK, -1>(sb + (u64)ib * SW, sa + (u64)ia * SW, 0);
    if (KEYS_ONLY) {
      // keys (time advanced) from the tile, the rest of the row from global memory, word by word
      const u64* k = take_a ? sa + (u64)ia * SW : sb + (u64)ib * SW;
      const u64* g = take_a ? A + (a0 + ia) * NW : B + (b0 + ib) * NW;
      u64* dst = out + (diag0 + o) * NW;
#pragma unroll
      for (int w = 0; w < SW; ++w) dst[w] = k[w];
      for (int w = SW; w < NW; ++w) dst[w] = g[w];
    } else {
      const u64* src = take_a ? sa + (u64)ia * SW : sb + (u64)ib * SW;
      u64 r[NW];
#pragma unroll
      for (int w = 0; w < NW; ++w) r[w] = src[w];
      store_row<NW>(out, diag0 + o, r);
    }
    if (take_a)
      ++ia;
    else
      ++ib;
  }
}

template <int RB>
int32_t merge_t(mzgpu_ctx* ctx, const u64* A, u64 na, const u64* B, u64 nb, u64 since, DevMem* out,
                u64* n_out) {
  constexpr u64 TILE = MergeCfg<RB>::TILE;
  const u64 n = na + nb;
  *n_out = 0;
  MZ_TRY(out->alloc(ctx, n * RB));
  if (n == 0) return MZGPU_OK;
  const u64 n_tiles = (n + TILE - 1) / TILE;
  DevMem split, merged;
  MZ_TRY(split.alloc(ctx, (n_tiles + 1) * 8));
  MZ_TRY(merged.alloc(ctx, n * RB));
  MZ_LAUNCH(ctx, (k_merge_partition<RB>), (unsigned)((n_tiles + 1 + 255) / 256), 256, 0, A, na, B, nb,
            since, n_tiles, split.as<u64>());
  MZ_BYTES(ctx, n * 2 * RB);
  MZ_LAUNCH(ctx, (k_merge_tiles<RB>), (unsigned)n_tiles, MT, 0, A, na, B, nb, since, split.as<u64>(),
            merged.as<u64>());
  MZ_TRY(mz_consolidate_sorted(ctx, RB, merged.p, n, out->p, n_out));
  return MZGPU_OK;
}

// ---------------------------------------------------------------- extract
template <int RB>
__global__ void __launch_bounds__(512) k_extract_count(const u64* __restrict__ rows, u64 n, u64 upper,
                                                       u32* __restrict__ tile_counts,
                                                       u64* __restrict__ min_keep) {
  constexpr int NW = RowT<RB>::NW, TW = RowT<RB>::TW;
  __shared__ u32 sm[34];
  u64 i = (u64)blockIdx.x * 512 + threadIdx.x;
  u32 ship = 0;
  u64 kt = ~0ull;
  if (i < n) {
    u64 t = rows[i * NW + (TW >= 0 ? TW : 0)];
    ship = t < upper ? 1u : 0u;
    if (!ship) kt = t;
  }
  u32 total;
  block_exclusive_scan(ship, sm, &total);
  if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    u64 o = __shfl_xor_sync(0xffffffffu, kt, off);
    kt = o < kt ? o : kt;
  }
  if (lane_id() == 0 && kt != ~0ull) atomicMin((unsigned long long*)min_keep, (unsigned long long)kt);
}

template <int RB>
__global__ void __launch_bounds__(512) k_extract_scatter(const u64* __restrict__ rows, u64 n, u64 upper,
                                                         const u32* __restrict__ tile_base,
                                                         u64* __restrict__ ship, u64* __restrict__ keep) {
  constexpr int NW = RowT<RB>::NW, TW = RowT<RB>::TW;
  __shared__ u32 sm[34];
  u64 i = (u64)blockIdx.x * 512 + threadIdx.x;
  u32 s = 0;
  u64 r[NW];
  if (i < n) {
    load_row<NW>(rows, i, r);
    s = r[TW >= 0 ? TW : 0] < upper ? 1u : 0u;
  }
  u32 total;
  u32 ex = block_exclusive_scan(s, sm, &total);
  if (i < n) {
    u64 ship_pos = (u64)tile_base[blockIdx.x] + ex;
    if (s)
      store_row<NW>(ship, ship_pos, r);
    else
      store_row<NW>(keep, i - ship_pos, r);
  }
}

template <int RB>
int32_t extract_t(mzgpu_ctx* ctx, const u64* rows, u64 n, u64 upper, DevMem* ship, u64* n_ship,
                  DevMem* keep, u64* n_keep, u64* min_keep_time) {
  *n_ship = 0;
  *n_keep = 0;
  *min_keep_time = MZGPU_FRONTIER_EMPTY;
  MZ_TRY(ship->alloc(ctx, n * RB));
  MZ_TRY(keep->alloc(ctx, n * RB));
  if (n == 0) return MZGPU_OK;
  const u64 n_tiles = (n + 511) / 512;
  DevMem tiles;
  MZ_TRY(tiles.alloc(ctx, n_tiles * 4));
  u64* d_total = ctx->d_scratch + 20;
  u64* d_min = ctx->d_scratch + 21;
  MZ_CUDA(ctx, cudaMemsetAsync(d_min, 0xff, 8, ctx->stream));
  MZ_LAUNCH(ctx, (k_extract_count<RB>), (unsigned)n_tiles, 512, 0, rows, n, upper, tiles.as<u32>(),
            d_min);
  MZ_LAUNCH(ctx, k_scan_tiles, 1, 1024, 0, tiles.as<u32>(), n_tiles, d_total);
  MZ_LAUNCH(ctx, (k_extract_scatter<RB>), (unsigned)n_tiles, 512, 0, rows, n, upper, tiles.as<u32>(),
            ship->as<u64>(), keep->as<u64>());
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 20, d_total, 16, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 16;
  *n_ship = ctx->h_scratch[20];
  *n_keep = n - *n_ship;
  *min_keep_time = ctx->h_scratch[21];
  return MZGPU_OK;
}

}  // namespace

int32_t mz_merge_consolidate(mzgpu_ctx* ctx, int row_bytes, const void* d_a, u64 na, const void* d_b,
                             u64 nb, u64 since, DevMem* out, u64* n_out) {
  return mz_dispatch<BatchWidths>(ctx, row_bytes, "merge", [&](auto RB) {
    return merge_t<RB>(ctx, (const u64*)d_a, na, (const u64*)d_b, nb, since, out, n_out);
  });
}

int32_t mz_extract(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, u64 upper, DevMem* ship,
                   u64* n_ship, DevMem* keep, u64* n_keep, u64* min_keep_time) {
  return mz_dispatch<BatchWidths>(ctx, row_bytes, "extract", [&](auto RB) {
    return extract_t<RB>(ctx, (const u64*)d_rows, n, upper, ship, n_ship, keep, n_keep, min_keep_time);
  });
}
