// consolidate.cu — the sweep half of consolidation (SURVEY.md a1):
// "sum diffs of equal (data, time) neighbours, drop zeros, truncate".
//
// Reference: the fold loop of Chunker::push_into
// (src/timely-util/src/columnar/batcher.rs:82-117) and the reference model
// consolidate() (:1116-1130); differential_dataflow::consolidation (external).
//
// On the GPU the sweep is a segmented sum over the sorted array:
//   k_heads   flags the first row of every run of equal keys, counts per tile
//   (scan)    tile bases
//   k_segsum  warp-segmented shuffle scan of the diff words, one atomic per
//             (warp, segment) into the segment accumulator (skew-robust: a hot
//             key costs one atomic per warp, never a per-key thread)
//   k_nz      flags segments with a non-zero sum, counts per tile
//   (scan)
//   k_emit    writes the surviving (key words, summed diff) rows, compacted
#include "common.cuh"

namespace {

constexpr int CT = 512;  // rows per tile == threads per block

template <int NW, int NK>
__device__ __forceinline__ bool key_differs(const u64* __restrict__ rows, u64 i) {
  const u64* a = rows + i * NW;
  const u64* b = a - NW;
  bool ne = false;
#pragma unroll
  for (int k = 0; k < NK; ++k) ne |= a[k] != b[k];
  return ne;
}

template <int NW, int NK>
__global__ void __launch_bounds__(CT) k_heads(const u64* __restrict__ rows, u64 n,
                                              u32* __restrict__ tile_counts) {
  __shared__ u32 sm[34];
  u64 i = (u64)blockIdx.x * CT + threadIdx.x;
  u32 flag = 0;
  if (i < n) flag = (i == 0) ? 1u : (key_differs<NW, NK>(rows, i) ? 1u : 0u);
  u32 total;
  block_exclusive_scan(flag, sm, &total);
  if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
}

template <int ND, int SG>
__device__ __forceinline__ void atomic_diff_add(u64* __restrict__ acc, const u64* d) {
  if (SG == MZ_SG_MAX) {
    atomic_diff_max<ND>(acc, d);
  } else if (ND == 8) {
    if (d[0]) atomicAdd((unsigned long long*)&acc[0], (unsigned long long)d[0]);
    if (d[1]) atomicAdd((unsigned long long*)&acc[1], (unsigned long long)d[1]);
    // 128-bit add: the atomic that wraps the low word carries into the high word
    u64 old = atomicAdd((unsigned long long*)&acc[2], (unsigned long long)d[2]);
    u64 carry = (old + d[2]) < old ? 1 : 0;
    u64 hi = d[3] + carry;
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

template <int NW, int NK, int ND>
__global__ void __launch_bounds__(CT) k_segsum(const u64* __restrict__ rows, u64 n,
                                               const u32* __restrict__ tile_base,
                                               u64* __restrict__ seg_sums,
                                               u32* __restrict__ seg_first) {
  constexpr int SG = RowT<NW * 8>::SG;
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * CT + threadIdx.x;
  const u32 lane = lane_id();
  const bool valid = i < n;
  u32 flag = 0;
  if (valid) flag = (i == 0) ? 1u : (key_differs<NW, NK>(rows, i) ? 1u : 0u);
  u32 total;
  u32 ex = block_exclusive_scan(flag, sm, &total);
  // segment id of row i = (#heads in [0, i]) - 1
  u32 seg = valid ? tile_base[blockIdx.x] + ex + flag - 1 : 0xffffffffu;
  u64 d[ND];
#pragma unroll
  for (int w = 0; w < ND; ++w) d[w] = valid ? rows[i * NW + NK + w] : 0;
  if (valid && flag) seg_first[seg] = (u32)i;
  // warp-segmented inclusive scan (segments are contiguous because rows are sorted)
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    u32 oseg = __shfl_up_sync(0xffffffffu, seg, off);
    u64 o[ND];
#pragma unroll
    for (int w = 0; w < ND; ++w) o[w] = __shfl_up_sync(0xffffffffu, d[w], off);
    if (lane >= (u32)off && oseg == seg) diff_add<ND, SG>(d, o);
  }
  u32 nseg = __shfl_down_sync(0xffffffffu, seg, 1);
  bool tail = valid && (lane == 31 || nseg != seg);
  if (tail) atomic_diff_add<ND, SG>(seg_sums + (u64)seg * ND, d);
}

template <int ND, int SG>
__global__ void __launch_bounds__(CT) k_nz(const u64* __restrict__ seg_sums,
                                           const u64* __restrict__ n_seg_ptr,
                                           u32* __restrict__ tile_counts) {
  __shared__ u32 sm[34];
  const u64 S = *n_seg_ptr;
  u64 s = (u64)blockIdx.x * CT + threadIdx.x;
  u32 flag = 0;
  if (s < S) flag = diff_is_zero<ND, SG>(seg_sums + s * ND) ? 0u : 1u;
  u32 total;
  block_exclusive_scan(flag, sm, &total);
  if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
}

template <int NW, int NK, int ND>
__global__ void __launch_bounds__(CT) k_emit(const u64* __restrict__ rows,
                                             const u64* __restrict__ seg_sums,
                                             const u32* __restrict__ seg_first,
                                             const u64* __restrict__ n_seg_ptr,
                                             const u32* __restrict__ tile_base,
                                             u64* __restrict__ out) {
  constexpr int SG = RowT<NW * 8>::SG;
  __shared__ u32 sm[34];
  const u64 S = *n_seg_ptr;
  u64 s = (u64)blockIdx.x * CT + threadIdx.x;
  u32 flag = 0;
  if (s < S) flag = diff_is_zero<ND, SG>(seg_sums + s * ND) ? 0u : 1u;
  u32 total;
  u32 ex = block_exclusive_scan(flag, sm, &total);
  if (flag) {
    u64 pos = (u64)tile_base[blockIdx.x] + ex;
    u64 r[NW];
    load_row<NW>(rows, seg_first[s], r);
#pragma unroll
    for (int w = 0; w < ND; ++w) r[NK + w] = seg_sums[s * ND + w];
    store_row<NW>(out, pos, r);
  }
}

template <int NW>
__global__ void __launch_bounds__(256) k_gather(const u64* __restrict__ rows,
                                                const u32* __restrict__ perm, u64 n,
                                                u64* __restrict__ out) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u64 r[NW];
  load_row<NW>(rows, perm[i], r);
  store_row<NW>(out, i, r);
}

template <int RB>
int32_t consolidate_sorted_t(mzgpu_ctx* ctx, const u64* rows, u64 n, u64* out, u64* n_out) {
  constexpr int NW = RowT<RB>::NW, NK = RowT<RB>::NK, ND = RowT<RB>::ND;
  *n_out = 0;
  if (n == 0) return MZGPU_OK;
  const u64 n_tiles = (n + CT - 1) / CT;
  DevMem tiles, seg_sums, seg_first;
  MZ_TRY(tiles.alloc(ctx, n_tiles * 4));
  MZ_TRY(seg_sums.alloc(ctx, n * 8 * ND));
  MZ_TRY(seg_first.alloc(ctx, n * 4));
  u64* d_nseg = ctx->d_scratch + 16;
  u64* d_nout = ctx->d_scratch + 17;
  MZ_CUDA(ctx, cudaMemsetAsync(seg_sums.p, 0, n * 8 * ND, ctx->stream));
  MZ_BYTES(ctx, n * NK * 8);
  MZ_LAUNCH(ctx, (k_heads<NW, NK>), (unsigned)n_tiles, CT, 0, rows, n, tiles.as<u32>());
  MZ_LAUNCH(ctx, k_scan_tiles, 1, 1024, 0, tiles.as<u32>(), n_tiles, d_nseg);
  MZ_BYTES(ctx, n * (NW * 8 + 4));
  MZ_LAUNCH(ctx, (k_segsum<NW, NK, ND>), (unsigned)n_tiles, CT, 0, rows, n, tiles.as<u32>(),
            seg_sums.as<u64>(), seg_first.as<u32>());
  MZ_LAUNCH(ctx, (k_nz<ND, RowT<RB>::SG>), (unsigned)n_tiles, CT, 0, seg_sums.as<u64>(), d_nseg, tiles.as<u32>());
  MZ_LAUNCH(ctx, k_scan_tiles, 1, 1024, 0, tiles.as<u32>(), n_tiles, d_nout);
  MZ_LAUNCH(ctx, (k_emit<NW, NK, ND>), (unsigned)n_tiles, CT, 0, rows, seg_sums.as<u64>(),
            seg_first.as<u32>(), d_nseg, tiles.as<u32>(), out);
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 16, d_nseg, 16, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 16;
  *n_out = ctx->h_scratch[17];
  return MZGPU_OK;
}

template <int RB>
int32_t gather_t(mzgpu_ctx* ctx, const u64* rows, const u32* perm, u64 n, u64* out) {
  constexpr int NW = RowT<RB>::NW;
  if (n == 0) return MZGPU_OK;
  MZ_BYTES(ctx, n * (4 + 2 * NW * 8));
  MZ_LAUNCH(ctx, (k_gather<NW>), (unsigned)((n + 255) / 256), 256, 0, rows, perm, n, out);
  return MZGPU_OK;
}

}  // namespace

int32_t mz_gather_rows(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, const u32* d_perm, u64 n,
                       void* d_out) {
  return mz_dispatch<RowWidths>(ctx, row_bytes, "gather", [&](auto RB) {
    return gather_t<RB>(ctx, (const u64*)d_rows, d_perm, n, (u64*)d_out);
  });
}

int32_t mz_consolidate_sorted(mzgpu_ctx* ctx, int row_bytes, const void* d_sorted, u64 n, void* d_out,
                              u64* n_out) {
  return mz_dispatch<RowWidths>(ctx, row_bytes, "consolidate", [&](auto RB) {
    return consolidate_sorted_t<RB>(ctx, (const u64*)d_sorted, n, (u64*)d_out, n_out);
  });
}

int32_t mz_sort_consolidate(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, DevMem* out,
                            u64* n_out) {
  *n_out = 0;
  MZ_TRY(out->alloc(ctx, n * (u64)row_bytes));
  if (n == 0) return MZGPU_OK;
  DevMem perm, sorted;
  MZ_TRY(mz_sort_perm(ctx, row_bytes, d_rows, n, &perm));
  MZ_TRY(sorted.alloc(ctx, n * (u64)row_bytes));
  MZ_TRY(mz_gather_rows(ctx, row_bytes, d_rows, perm.as<u32>(), n, sorted.p));
  MZ_TRY(mz_consolidate_sorted(ctx, row_bytes, sorted.p, n, out->p, n_out));
  return MZGPU_OK;
}
