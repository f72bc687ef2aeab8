// index.cu — per-batch open-addressing hash index over distinct keys
// (SURVEY.md a5/a8).
//
// The reference's OrdValBatch keeps a sorted `keys[]` array and its cursor
// finds a key with exponential + binary search (`seek_key`; usage
// src/compute/src/render/join/mz_join_core.rs:606-621).  On the GPU a probe is
// one 128-bit load of a 16-byte slot {key, first row + 1} (linear probing, load
// factor <= 0.5), after which the key's updates are a contiguous run of the
// batch's sorted rows.
#include "common.cuh"

namespace {

template <int NW>
__global__ void __launch_bounds__(512) k_count_keys(const u64* __restrict__ rows, u64 n,
                                                    unsigned long long* __restrict__ count) {
  u64 i = (u64)blockIdx.x * 512 + threadIdx.x;
  bool head = false;
  if (i < n) head = (i == 0) || rows[i * NW] != rows[(i - 1) * NW];
  // one atomic pair per CTA: same-address atomics from every warp serialise in L2
  __shared__ u32 s_heads[16], s_run[16];
  const u32 m = __ballot_sync(0xffffffffu, head);
  // longest run of one key (saturating at 1024): bounds the fan-out of a probe
  u32 run = 0;
  if (head) {
    const u64 key = rows[i * NW];
    run = 1;
    while (run < 1024 && i + run < n && rows[(i + run) * NW] == key) ++run;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    u32 o = __shfl_xor_sync(0xffffffffu, run, off);
    run = o > run ? o : run;
  }
  if (lane_id() == 0) {
    s_heads[threadIdx.x >> 5] = __popc(m);
    s_run[threadIdx.x >> 5] = run;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    u32 h = threadIdx.x < 16 ? s_heads[threadIdx.x] : 0;
    u32 r = threadIdx.x < 16 ? s_run[threadIdx.x] : 0;
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) {
      h += __shfl_xor_sync(0xffffffffu, h, off);
      u32 o = __shfl_xor_sync(0xffffffffu, r, off);
      r = o > r ? o : r;
    }
    if (threadIdx.x == 0 && h) {
      atomicAdd(count, (unsigned long long)h);
      atomicMax(count + 1, (unsigned long long)r);
    }
  }
}

template <int NW>
__global__ void __launch_bounds__(512) k_build_index(const u64* __restrict__ rows, u64 n,
                                                     HashSlot* __restrict__ table, u64 mask) {
  u64 i = (u64)blockIdx.x * 512 + threadIdx.x;
  if (i >= n) return;
  u64 key = rows[i * NW];
  if (i != 0 && rows[(i - 1) * NW] == key) return;
  // the key's run length, if it ends within 64 rows (longer runs are left for the reader to scan)
  u64 run = 1;
  while (run <= 64 && i + run < n && rows[(i + run) * NW] == key) ++run;
  const u64 meta = (i + 1) | ((run <= 64 ? run : 0ull) << 44);
  u64 h = mix64(key) & mask;
  while (true) {
    // distinct keys only: claim the first empty slot
    unsigned long long prev = atomicCAS((unsigned long long*)&table[h].meta, 0ull, (unsigned long long)meta);
    if (prev == 0ull) {
      table[h].key = key;
      return;
    }
    h = (h + 1) & mask;
  }
}


// ---- Cursor::seek_key, batched (a8): one thread per probe key, binary search for the first row
// whose key is >= the probe key (exactly seek_key's position: mz_join_core.rs:606-621 walks two
// cursors with seek_key / step_key), then the end of that key's run.  out[i] = {key found, first
// row, rows of that key}; len == 0 means the cursor ran off the end (key_valid() == false).
template <int NW>
__global__ void __launch_bounds__(256) k_seek_keys(const u64* __restrict__ rows, const DLen dn,
                                                   const u64* __restrict__ probe, u64 n_probe,
                                                   u64* __restrict__ out /* [n_probe][3] */) {
  const u64 n = dlen_get(dn);
  const u64 i = (u64)blockIdx.x * 256 + threadIdx.x;
  if (i >= n_probe) return;
  const u64 k = probe[i];
  u64 lo = 0, hi = n;
  while (lo < hi) {
    const u64 mid = (lo + hi) >> 1;
    if (rows[mid * NW] < k)
      lo = mid + 1;
    else
      hi = mid;
  }
  u64 found = 0, len = 0;
  if (lo < n) {
    found = rows[lo * NW];
    // end of the run: first row whose key is greater
    u64 l2 = lo + 1, h2 = n;
    while (l2 < h2) {
      const u64 mid = (l2 + h2) >> 1;
      if (rows[mid * NW] <= found)
        l2 = mid + 1;
      else
        h2 = mid;
    }
    len = l2 - lo;
  }
  out[i * 3 + 0] = found;
  out[i * 3 + 1] = lo;
  out[i * 3 + 2] = len;
}

// ---- Cursor::step_key over the whole batch, in pages: the distinct keys with ordinal in
// [first_ordinal, first_ordinal + max) and their runs.  Heads are found by comparison with the
// previous row; their ordinals by a block scan + look-back-free two-step (count per tile, scan).
template <int NW>
__global__ void __launch_bounds__(256) k_key_heads_count(const u64* __restrict__ rows, const DLen dn,
                                                         u32* __restrict__ tile_counts) {
  __shared__ u32 sm[34];
  const u64 n = dlen_get(dn);
  const u64 i = (u64)blockIdx.x * 256 + threadIdx.x;
  const u32 head = (i < n && (i == 0 || rows[i * NW] != rows[(i - 1) * NW])) ? 1u : 0u;
  u32 total;
  block_exclusive_scan(head, sm, &total);
  if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
}
template <int NW>
__global__ void __launch_bounds__(256) k_key_heads_emit(const u64* __restrict__ rows, const DLen dn,
                                                        const u32* __restrict__ tile_base, u64 first_ordinal,
                                                        u64 max_keys, u64* __restrict__ out /* [max][3] */) {
  __shared__ u32 sm[34];
  const u64 n = dlen_get(dn);
  const u64 i = (u64)blockIdx.x * 256 + threadIdx.x;
  const u32 head = (i < n && (i == 0 || rows[i * NW] != rows[(i - 1) * NW])) ? 1u : 0u;
  u32 total;
  const u32 ex = block_exclusive_scan(head, sm, &total);
  if (!head) return;
  const u64 ord = (u64)tile_base[blockIdx.x] + ex;
  if (ord < first_ordinal || ord >= first_ordinal + max_keys) return;
  const u64 key = rows[i * NW];
  u64 e = i + 1;
  while (e < n && rows[e * NW] == key) ++e;
  u64* o = out + (ord - first_ordinal) * 3;
  o[0] = key;
  o[1] = i;
  o[2] = e - i;
}

}  // namespace

int32_t mz_count_keys(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, u64* n_keys, u64* max_run) {
  *n_keys = 0;
  *max_run = 0;
  if (n == 0) return MZGPU_OK;
  u64* d_count = ctx->d_scratch + 24;
  MZ_CUDA(ctx, cudaMemsetAsync(d_count, 0, 16, ctx->stream));
  unsigned grid = (unsigned)((n + 511) / 512);
  MZ_TRY(mz_dispatch<BatchWidths>(ctx, row_bytes, "index", [&](auto RB) {
    MZ_LAUNCH(ctx, k_count_keys<RowT<RB>::NW>, grid, 512, 0, (const u64*)d_rows, n, (unsigned long long*)d_count);
    return MZGPU_OK;
  }));
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 24, d_count, 16, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 16;
  *n_keys = ctx->h_scratch[24];
  *max_run = ctx->h_scratch[25];
  return MZGPU_OK;
}

int32_t mz_build_index(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, u64 n_keys,
                       DevMem* table, u64* table_slots) {
  u64 slots = 2;
  while (slots < 2 * n_keys) slots <<= 1;
  *table_slots = slots;
  MZ_TRY(table->alloc(ctx, slots * sizeof(HashSlot)));
  MZ_CUDA(ctx, cudaMemsetAsync(table->p, 0, slots * sizeof(HashSlot), ctx->stream));
  if (n == 0) return MZGPU_OK;
  unsigned grid = (unsigned)((n + 511) / 512);
  return mz_dispatch<BatchWidths>(ctx, row_bytes, "index", [&](auto RB) {
    MZ_LAUNCH(ctx, k_build_index<RowT<RB>::NW>, grid, 512, 0, (const u64*)d_rows, n, table->as<HashSlot>(), slots - 1);
    return MZGPU_OK;
  });
}

// a8: batched seek_key.  d_probe: n_probe keys (device); d_out: n_probe x {key, first, len}.
int32_t mz_seek_keys(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, DLen n, const u64* d_probe, u64 n_probe,
                     u64* d_out) {
  if (n_probe == 0) return MZGPU_OK;
  unsigned grid = (unsigned)((n_probe + 255) / 256);
  return mz_dispatch<BatchWidths>(ctx, row_bytes, "seek_keys", [&](auto RB) {
    MZ_LAUNCH(ctx, k_seek_keys<RowT<RB>::NW>, grid, 256, 0, (const u64*)d_rows, n, d_probe, n_probe, d_out);
    return MZGPU_OK;
  });
}

// a8: step_key paging.  n_rows is exact (the caller resolved the batch); d_out: max_keys x {key, first, len}.
int32_t mz_key_page(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n_rows, u64 first_ordinal, u64 max_keys,
                    u64* d_out) {
  if (n_rows == 0 || max_keys == 0) return MZGPU_OK;
  const u64 tiles = (n_rows + 255) / 256;
  DevMem counts;
  MZ_TRY(counts.alloc(ctx, tiles * 4 + 16));
  DevMem total;
  MZ_TRY(total.alloc(ctx, 16));
  const u64* r = (const u64*)d_rows;
  const DLen dn = dlen_imm(n_rows);
  return mz_dispatch<BatchWidths>(ctx, row_bytes, "key_page", [&](auto RB) {
    constexpr int NW = RowT<RB>::NW;
    MZ_LAUNCH(ctx, k_key_heads_count<NW>, (unsigned)tiles, 256, 0, r, dn, counts.as<u32>());
    MZ_LAUNCH(ctx, k_scan_tiles, 1, 1024, 0, counts.as<u32>(), tiles, total.as<u64>());
    MZ_LAUNCH(ctx, k_key_heads_emit<NW>, (unsigned)tiles, 256, 0, r, dn, counts.as<u32>(), first_ordinal, max_keys,
              d_out);
    return MZGPU_OK;
  });
}
