// radix.cuh — one tile of one 8-bit LSD radix pass ("onesweep" with decoupled
// look-back), shared by the stand-alone pass kernel (sort.cu) and the fused
// cooperative small-input kernel (fused.cu).
#pragma once
#include "common.cuh"

constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr u32 RS_FLAG_PARTIAL = 1u << 30;
constexpr u32 RS_FLAG_INCLUSIVE = 2u << 30;
constexpr u32 RS_VALUE_MASK = (1u << 30) - 1;

template <int ITEMS, int THREADS = RS_THREADS>
struct RsSmemT {
  alignas(16) u64 keys[THREADS * ITEMS];
  alignas(16) u32 vals[THREADS * ITEMS];
  alignas(8) u64 mbar;  // TMA tile load: transaction barrier
  u32 whist[THREADS / 32][256];
  u32 digit_start[256];
  u32 gofs[256];
  u32 scan[34];
  u32 tile;
};

// Sort tile `tile` (RS_THREADS*ITEMS consecutive (key, val) pairs) by digit
// (key >> shift) & 255 into (kout, vout).  Stable.  Requirements: blockDim.x ==
// RS_THREADS; tiles are processed so that every tile < `tile` is already done or
// is being processed by a co-resident CTA (look-back progress); tile_state is
// zero before the pass.  No __restrict__ here: inside the fused kernel the
// input of one pass was written by other CTAs in the previous phase.  Ends with a __syncthreads(): `s` can be reused.
// tile-state words are read and written with GPU-scope relaxed accesses (a word
// carries its own flag, so no ordering with other data is needed)
__device__ __forceinline__ u32 rs_load(const u32* p) {
  u32 v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void rs_store(u32* p, u32 v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// lanes of the warp whose 8-bit digit equals this lane's: eight ballots.  (The
// hardware MATCH.ANY runs on the address-divergence unit at a small fraction of
// the ballot rate: with ~30 distinct digits per warp it becomes the pipe that
// bounds the whole pass.)
__device__ __forceinline__ u32 match_digit(u32 d) {
  u32 m = 0xffffffffu;
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    const bool bit = (d >> b) & 1u;
    const u32 bal = __ballot_sync(0xffffffffu, bit);
    m &= bit ? bal : ~bal;
  }
  return m;
}

// ---- TMA (bulk async copy) helpers: one thread arms a transaction barrier with the tile's byte
// count and issues cp.async.bulk global -> shared; everybody waits on the barrier's phase.
__device__ __forceinline__ u32 rs_smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void rs_mbar_init(u64* bar, u32 count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(rs_smem_addr(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void rs_mbar_expect_tx(u64* bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(rs_smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void rs_bulk_g2s(void* dst_smem, const void* src_gmem, u32 bytes, u64* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   rs_smem_addr(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(rs_smem_addr(bar))
               : "memory");
}
__device__ __forceinline__ void rs_mbar_wait(u64* bar, u32 parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(rs_smem_addr(bar)),
      "r"(parity)
      : "memory");
}

template <int ITEMS, int THREADS = RS_THREADS, bool TMA_LOAD = false>
__device__ __forceinline__ void rs_tile_pass(RsSmemT<ITEMS, THREADS>& s, u32 tile, const u64* kin,
                                             const u32* vin, u64* kout,
                                             u32* vout, u64 n, int shift,
                                             const u32* gbase, u32* tile_state) {
  constexpr u32 TILE = THREADS * ITEMS;
  constexpr int WARPS = THREADS / 32;
  const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const u64 base = (u64)tile * TILE;
  const u32 n_valid = (u32)((n - base) < (u64)TILE ? (n - base) : (u64)TILE);
  // TMA-staged tile load (full tiles): ONE thread issues two bulk copies (keys, values) into the
  // staging arrays and the whole tile arrives through the async proxy while the CTA clears its
  // histograms; the partial last tile takes ordinary loads.
  const bool tma = TMA_LOAD && n_valid == TILE;
  if (TMA_LOAD) {
    if (tid == 0) rs_mbar_init(&s.mbar, 1);
    __syncthreads();
    if (tma && tid == 0) {
      rs_mbar_expect_tx(&s.mbar, TILE * 12u);
      rs_bulk_g2s(s.keys, kin + base, TILE * 8u, &s.mbar);
      rs_bulk_g2s(s.vals, vin + base, TILE * 4u, &s.mbar);
    }
  }
  for (int i = tid; i < WARPS * 256; i += THREADS) (&s.whist[0][0])[i] = 0;
  __syncthreads();

  // warp-striped load: element index inside the tile = warp*(ITEMS*32) + j*32 + lane
  u64 key[ITEMS];
  u32 val[ITEMS];
  u32 rank[ITEMS];
  const u32 wb = warp * (ITEMS * 32);
  if (tma) {
    rs_mbar_wait(&s.mbar, 0);
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
      const u32 idx = wb + j * 32 + lane;
      key[j] = s.keys[idx];
      val[j] = s.vals[idx];
    }
  } else {
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
      u32 idx = wb + j * 32 + lane;
      bool ok = idx < n_valid;
      key[j] = ok ? kin[base + idx] : ~0ull;
      val[j] = ok ? vin[base + idx] : 0u;
    }
  }
  // stable in-warp ranking with match_digit / popc (warp-shuffle histograms)
  const u32 lt_mask = (1u << lane) - 1;
#pragma unroll
  for (int j = 0; j < ITEMS; ++j) {
    u32 d = (u32)((key[j] >> shift) & 255);
    u32 m = match_digit(d);
    u32 leader = __ffs(m) - 1;
    u32 old = 0;
    if (lane == leader) {
      old = s.whist[warp][d];
      s.whist[warp][d] = old + __popc(m);
    }
    old = __shfl_sync(0xffffffffu, old, leader);
    rank[j] = old + __popc(m & lt_mask);
    __syncwarp();
  }
  __syncthreads();

  // thread d owns digit d: exclusive scan across warps; the tile's digit counts
  // are published at once (successors only need this aggregate to move on)
  u32 my_tot_valid = 0;
  if (THREADS == 256 || tid < 256) {
    const u32 d = tid;
    u32 tot = 0;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) {
      u32 c = s.whist[w][d];
      s.whist[w][d] = tot;
      tot += c;
    }
    const u32 n_invalid = TILE - n_valid;  // padding keys all carry digit 255
    my_tot_valid = (d == 255) ? tot - n_invalid : tot;
    rs_store(&tile_state[(u64)tile * 256 + d], (tile == 0 ? RS_FLAG_INCLUSIVE : RS_FLAG_PARTIAL) | my_tot_valid);
    s.digit_start[d] = tot;  // digit totals; scanned below
  }
  __syncthreads();
  {
    // exclusive scan of the 256 digit totals (every thread of the CTA takes part in the barriers)
    u32 v = tid < 256 ? s.digit_start[tid] : 0;
    u32 total;
    u32 ds = block_exclusive_scan(v, s.scan, &total);
    if (tid < 256) s.digit_start[tid] = ds;
  }
  __syncthreads();

  // stage the tile in shared memory in digit order
#pragma unroll
  for (int j = 0; j < ITEMS; ++j) {
    u32 d = (u32)((key[j] >> shift) & 255);
    u32 pos = s.digit_start[d] + s.whist[warp][d] + rank[j];
    s.keys[pos] = key[j];
    s.vals[pos] = val[j];
  }
  // decoupled look-back, as late as possible (the predecessors have had the whole
  // staging step to publish) and four predecessors per round trip
  if (THREADS == 256 || tid < 256) {
    const u32 d = tid;
    u32 excl = 0;
    if (tile != 0) {
      long long t = (long long)tile - 1;
      bool done = false;
      while (!done) {
        u32 v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
          v[q] = (t - q >= 0) ? rs_load(&tile_state[(u64)(t - q) * 256 + d]) : RS_FLAG_INCLUSIVE;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const u32 flag = v[q] >> 30;
          if (flag == 0) {  // not published yet: re-read from here
            t -= q;
            break;
          }
          excl += v[q] & RS_VALUE_MASK;
          if (flag == 2) {
            done = true;
            break;
          }
          if (q == 3) t -= 4;
        }
      }
      rs_store(&tile_state[(u64)tile * 256 + d], RS_FLAG_INCLUSIVE | ((excl + my_tot_valid) & RS_VALUE_MASK));
    }
    s.gofs[d] = gbase[d] + excl - s.digit_start[d];  // global position = gofs[d] + local position
  }
  __syncthreads();
  // coalesced runs per digit
  for (u32 i = tid; i < n_valid; i += THREADS) {
    u64 k = s.keys[i];
    u32 d = (u32)((k >> shift) & 255);
    u32 g = s.gofs[d] + i;
    kout[g] = k;
    vout[g] = s.vals[i];
  }
  __syncthreads();
}
