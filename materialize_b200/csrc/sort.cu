// sort.cu — LSB radix sort of packed update rows (SURVEY.md a1/a2).
//
// Replaces the comparison sorts on the reference's hot path:
//   differential_dataflow::consolidation::consolidate_updates (sort by (data, time)),
//   callers src/compute/src/render/join/mz_join_core.rs:563, delta_join.rs:649
//   Chunker::push_into `permutation.sort()`  src/timely-util/src/columnar/batcher.rs:74-79
//   ColumnationChunker::form_chunk            src/timely-util/src/columnation.rs:477-488
//
// H100 design (HBM-bound integer work, no tensor-core path):
//   1. one pass over the rows finds min/max of every key word, so constant and
//      narrow words cost no radix passes (times are usually one value, keys a
//      few dozen bits);
//   2. the varying bits are packed into one 64-bit composite per row, carried
//      with a 32-bit row index: the sort moves 12 B per row per pass instead of
//      the 32..80 B row;
//   3. a single-read histogram kernel counts all digit places at once;
//   4. each 8-bit digit pass is ONE kernel ("onesweep"): tiles rank their keys
//      with warp match/shuffle histograms, resolve their global offsets with a
//      decoupled look-back over per-tile digit counts, stage the tile in shared
//      memory in digit order and write out coalesced runs;
//   5. rows are gathered once, by the final permutation (consolidate.cu).
#include "common.cuh"
#include "radix.cuh"

namespace {

// tile shape of the pass kernel: RS_ITEMS keys per thread, RS_THREADS threads, RS_MINB CTAs per SM
constexpr int RS_ITEMS = 16;
constexpr int RS_MINB = 3;

struct ChunkPlan {
  int nwords;
  int word[6];
  int shift[6];
  u64 minv[6];
};

// -------------------------------------------------------------- analyze
template <int NW, int NK>
__global__ void __launch_bounds__(256) k_analyze(const u64* __restrict__ rows, u64 n,
                                                 u64* __restrict__ minmax) {
  u64 mn[NK], mx[NK];
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    mn[k] = ~0ull;
    mx[k] = 0;
  }
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    const u64* p = rows + i * NW;
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      u64 v = p[k];
      mn[k] = v < mn[k] ? v : mn[k];
      mx[k] = v > mx[k] ? v : mx[k];
    }
  }
#pragma unroll
  for (int k = 0; k < NK; ++k) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      u64 a = __shfl_xor_sync(0xffffffffu, mn[k], off);
      u64 b = __shfl_xor_sync(0xffffffffu, mx[k], off);
      mn[k] = a < mn[k] ? a : mn[k];
      mx[k] = b > mx[k] ? b : mx[k];
    }
    if (lane_id() == 0) {
      atomicMin((unsigned long long*)&minmax[2 * k], (unsigned long long)mn[k]);
      atomicMax((unsigned long long*)&minmax[2 * k + 1], (unsigned long long)mx[k]);
    }
  }
}

__global__ void k_init_minmax(u64* minmax, int nk) {
  int i = threadIdx.x;
  if (i < nk) {
    minmax[2 * i] = ~0ull;
    minmax[2 * i + 1] = 0;
  }
}

// ------------------------------------------------------------------ pack
template <int NW>
__global__ void __launch_bounds__(256) k_pack(const u64* __restrict__ rows, const u32* __restrict__ perm,
                                              u64 n, ChunkPlan cp, u64* __restrict__ keys,
                                              u32* __restrict__ vals) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u32 src = perm != nullptr ? perm[i] : (u32)i;
  const u64* p = rows + (u64)src * NW;
  u64 c = 0;
  for (int j = 0; j < cp.nwords; ++j) c |= (p[cp.word[j]] - cp.minv[j]) << cp.shift[j];
  keys[i] = c;
  vals[i] = src;
}

__global__ void k_iota(u32* perm, u64 n) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) perm[i] = (u32)i;
}

// ------------------------------------------------- all-pass digit histogram
__global__ void __launch_bounds__(256) k_rs_hist(const u64* __restrict__ keys, u64 n, int npass,
                                                 u32* __restrict__ ghist) {
  __shared__ u32 sh[8 * 256];
  for (int i = threadIdx.x; i < npass * 256; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    u64 k = keys[i];
    for (int p = 0; p < npass; ++p) atomicAdd(&sh[p * 256 + (u32)((k >> (8 * p)) & 255)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < npass * 256; i += blockDim.x) {
    u32 v = sh[i];
    if (v) atomicAdd(&ghist[i], v);
  }
}

// exclusive scan of each pass's 256 bins -> global digit bases
__global__ void __launch_bounds__(256) k_rs_scan_hist(u32* __restrict__ ghist, int npass) {
  __shared__ u32 sm[33];
  for (int p = 0; p < npass; ++p) {
    u32 v = ghist[p * 256 + threadIdx.x];
    u32 total;
    u32 ex = block_exclusive_scan(v, sm, &total);
    ghist[p * 256 + threadIdx.x] = ex;
  }
}

// ------------------------------------------------------------ onesweep pass
template <int ITEMS, int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) k_rs_onesweep(
    const u64* __restrict__ kin, const u32* __restrict__ vin, u64* __restrict__ kout,
    u32* __restrict__ vout, u64 n, int shift, const u32* __restrict__ gbase,
    u32* __restrict__ tile_state, u32* __restrict__ tile_counter) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typedef RsSmemT<ITEMS, THREADS> Smem;
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  // dynamic tile assignment: tile t only starts after tiles < t have started,
  // which is what makes the look-back deadlock-free
  if (threadIdx.x == 0) s.tile = atomicAdd(tile_counter, 1u);
  __syncthreads();
  rs_tile_pass<ITEMS, THREADS, true>(s, s.tile, kin, vin, kout, vout, n, shift, gbase, tile_state);
}

static int32_t launch_onesweep(mzgpu_ctx* ctx, const u64* kin, const u32* vin, u64* kout, u32* vout, u64 n,
                               int shift, const u32* gbase, u32* state, u32* counter) {
  typedef RsSmemT<RS_ITEMS, RS_THREADS> Smem;
  static bool attr_set = false;
  if (!attr_set) {
    MZ_CUDA(ctx, cudaFuncSetAttribute(k_rs_onesweep<RS_ITEMS, RS_THREADS, RS_MINB>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem)));
    attr_set = true;
  }
  const u64 n_tiles = (n + (u64)RS_ITEMS * RS_THREADS - 1) / ((u64)RS_ITEMS * RS_THREADS);
  MZ_BYTES(ctx, n * 24);  // read key+idx (12 B), write key+idx (12 B)
  {
    ProfScope _prof(ctx, "k_rs_onesweep");
    k_rs_onesweep<RS_ITEMS, RS_THREADS, RS_MINB><<<(unsigned)n_tiles, RS_THREADS, sizeof(Smem), ctx->stream>>>(
        kin, vin, kout, vout, n, shift, gbase, state, counter);
  }
  ctx->stats.kernel_launches++;
  MZ_CUDA(ctx, cudaGetLastError());
  return MZGPU_OK;
}

static int bit_width_u64(u64 x) {
  int b = 0;
  while (x) {
    ++b;
    x >>= 1;
  }
  return b;
}

// Sort (keys, vals) pairs by the low `bits` bits of keys.  Result ends in
// (*k_cur, *v_cur) which alias either the a or the b buffers.
int32_t radix_sort_pairs(mzgpu_ctx* ctx, u64* ka, u32* va, u64* kb, u32* vb, u64 n, int bits,
                         u64** k_res, u32** v_res) {
  int npass = (bits + 7) / 8;
  *k_res = ka;
  *v_res = va;
  if (npass == 0 || n <= 1) return MZGPU_OK;
  const u64 tile = (u64)RS_ITEMS * RS_THREADS;
  const u64 n_tiles = (n + tile - 1) / tile;
  DevMem hist, state, counters;
  MZ_TRY(hist.alloc(ctx, (size_t)npass * 256 * 4));
  MZ_TRY(state.alloc(ctx, (size_t)npass * n_tiles * 256 * 4));
  MZ_TRY(counters.alloc(ctx, (size_t)npass * 4));
  MZ_CUDA(ctx, cudaMemsetAsync(hist.p, 0, hist.bytes, ctx->stream));
  MZ_CUDA(ctx, cudaMemsetAsync(state.p, 0, state.bytes, ctx->stream));
  MZ_CUDA(ctx, cudaMemsetAsync(counters.p, 0, counters.bytes, ctx->stream));
  {
    u64 blocks = (n + 256 * 16 - 1) / (256 * 16);
    u64 maxb = (u64)ctx->num_sms * 8;
    if (blocks > maxb) blocks = maxb;
    MZ_BYTES(ctx, n * 8);
    MZ_LAUNCH(ctx, k_rs_hist, (unsigned)blocks, 256, 0, ka, n, npass, hist.as<u32>());
    MZ_LAUNCH(ctx, k_rs_scan_hist, 1, 256, 0, hist.as<u32>(), npass);
  }
  u64 *kin = ka, *kout = kb;
  u32 *vin = va, *vout = vb;
  for (int p = 0; p < npass; ++p) {
    const u32* gb = hist.as<u32>() + p * 256;
    u32* stp = state.as<u32>() + (size_t)p * n_tiles * 256;
    u32* cnt = counters.as<u32>() + p;
    MZ_TRY(launch_onesweep(ctx, kin, vin, kout, vout, n, 8 * p, gb, stp, cnt));
    std::swap(kin, kout);
    std::swap(vin, vout);
  }
  *k_res = kin;
  *v_res = vin;
  return MZGPU_OK;
}

template <int RB>
int32_t sort_perm_t(mzgpu_ctx* ctx, const u64* d_rows, u64 n, DevMem* perm_out) {
  constexpr int NW = RowT<RB>::NW, NK = RowT<RB>::NK;
  if (n >= (1ull << 30)) {
    MZ_SET_ERR(ctx, "sort: %llu rows exceed the 2^30 per-call limit", (unsigned long long)n);
    return MZGPU_E_UNSUPPORTED;
  }
  MZ_TRY(perm_out->alloc(ctx, n * 4));
  if (n == 0) return MZGPU_OK;
  // 1. key ranges
  MZ_LAUNCH(ctx, k_init_minmax, 1, 32, 0, ctx->d_scratch, NK);
  {
    u64 blocks = (n + 255) / 256;
    u64 maxb = (u64)ctx->num_sms * 8;
    if (blocks > maxb) blocks = maxb;
    MZ_BYTES(ctx, n * NK * 8);
    MZ_LAUNCH(ctx, (k_analyze<NW, NK>), (unsigned)blocks, 256, 0, d_rows, n, ctx->d_scratch);
  }
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch, ctx->d_scratch, 2 * NK * 8, cudaMemcpyDeviceToHost,
                               ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 2 * NK * 8;
  for (int k = 0; k < 2 * NK; ++k) ctx->last_minmax[k] = ctx->h_scratch[k];
  ctx->last_minmax_valid = true;
  // 2. plan chunks of <= 64 composite bits, least significant word first
  int wbits[NK];
  u64 wmin[NK];
  int total_bits = 0;
  for (int k = 0; k < NK; ++k) {
    wmin[k] = ctx->h_scratch[2 * k];
    wbits[k] = bit_width_u64(ctx->h_scratch[2 * k + 1] - ctx->h_scratch[2 * k]);
    total_bits += wbits[k];
  }
  if (total_bits == 0) {
    MZ_LAUNCH(ctx, k_iota, (unsigned)((n + 255) / 256), 256, 0, perm_out->as<u32>(), n);
    return MZGPU_OK;
  }
  std::vector<ChunkPlan> chunks;
  {
    ChunkPlan cur;
    cur.nwords = 0;
    int used = 0;
    for (int k = NK - 1; k >= 0; --k) {
      if (wbits[k] == 0) continue;
      // (a chunk holds at most 6 words: only the 7-word TopK window rows can reach that)
      if (used + wbits[k] > 64 || cur.nwords == 6) {
        chunks.push_back(cur);
        cur.nwords = 0;
        used = 0;
      }
      cur.word[cur.nwords] = k;
      cur.shift[cur.nwords] = used;
      cur.minv[cur.nwords] = wmin[k];
      cur.nwords++;
      used += wbits[k];
    }
    if (cur.nwords > 0) chunks.push_back(cur);
  }
  // 3. one stable sort round per chunk
  DevMem ka, kb, va, vb;
  MZ_TRY(ka.alloc(ctx, n * 8));
  MZ_TRY(kb.alloc(ctx, n * 8));
  MZ_TRY(va.alloc(ctx, n * 4));
  MZ_TRY(vb.alloc(ctx, n * 4));
  const u32* perm = nullptr;
  u32* v_res = nullptr;
  for (size_t c = 0; c < chunks.size(); ++c) {
    int bits = 0;
    for (int j = 0; j < chunks[c].nwords; ++j) {
      int k = chunks[c].word[j];
      bits = chunks[c].shift[j] + wbits[k];
    }
    // pack into (ka, va); if the previous round's result lives in va, pack into (kb, vb)
    u64* kdst = ka.as<u64>();
    u32* vdst = va.as<u32>();
    u64* kalt = kb.as<u64>();
    u32* valt = vb.as<u32>();
    if (perm == va.as<u32>()) {
      std::swap(kdst, kalt);
      std::swap(vdst, valt);
    }
    MZ_BYTES(ctx, n * (chunks[c].nwords * 8 + 12 + (perm ? 4 : 0)));
    MZ_LAUNCH(ctx, (k_pack<NW>), (unsigned)((n + 255) / 256), 256, 0, d_rows, perm, n, chunks[c], kdst,
              vdst);
    u64* k_res;
    MZ_TRY(radix_sort_pairs(ctx, kdst, vdst, kalt, valt, n, bits, &k_res, &v_res));
    perm = v_res;
  }
  MZ_CUDA(ctx, cudaMemcpyAsync(perm_out->p, v_res, n * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  return MZGPU_OK;
}

}  // namespace

int32_t mz_sort_perm(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, u64 n, DevMem* perm_out) {
  return mz_dispatch<RowWidths>(ctx, row_bytes, "sort",
                                [&](auto RB) { return sort_perm_t<RB>(ctx, (const u64*)d_rows, n, perm_out); });
}
