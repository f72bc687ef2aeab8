// exchange.cu — the Exchange pact as a partition kernel (SURVEY.md a13, §8e).
//
// Reference: timely `Exchange(|k| k.hashed())` before every stateful operator
// (src/compute/src/extensions/arrange.rs:116, src/timely-util/src/columnar.rs:227-237,
// half_join's internal exchange).  Routing = FNV-1a 64 of the key's 8 LE bytes
// (Hashable::hashed in DD 0.23) modulo peers; output collections do not depend
// on the routing function.
//
// Rows are bucketed by destination on the device (count -> offsets -> scatter
// with one global atomic per (CTA, destination)); mzgpu_exchange (host.cu) then
// moves the buckets with one grouped ncclSend/ncclRecv all-to-all over NVLink.
#include "common.cuh"

namespace {

constexpr int XT = 256;
constexpr int MAX_PEERS = 64;

__host__ __device__ __forceinline__ u64 fnv1a64(u64 key) {
  u64 h = 0xcbf29ce484222325ull;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    h ^= (key >> (8 * i)) & 0xff;
    h *= 0x100000001b3ull;
  }
  return h;
}

template <int NW>
__global__ void __launch_bounds__(XT) k_part_count(const u64* __restrict__ rows, const DLen dn, u32 peers,
                                                   unsigned long long* __restrict__ counts) {
  const u64 n = dlen_get(dn);
  __shared__ u32 sh[MAX_PEERS];
  if (threadIdx.x < MAX_PEERS) sh[threadIdx.x] = 0;
  __syncthreads();
  for (u64 i = (u64)blockIdx.x * XT + threadIdx.x; i < n; i += (u64)gridDim.x * XT)
    atomicAdd(&sh[(u32)(fnv1a64(rows[i * NW]) % peers)], 1u);
  __syncthreads();
  if (threadIdx.x < peers && sh[threadIdx.x]) atomicAdd(&counts[threadIdx.x], (unsigned long long)sh[threadIdx.x]);
}

template <int NW>
__global__ void __launch_bounds__(XT) k_part_scatter(const u64* __restrict__ rows, const DLen dn, u32 peers,
                                                     unsigned long long* __restrict__ cursors,
                                                     u64* __restrict__ out) {
  const u64 n = dlen_get(dn);
  __shared__ u32 sh_count[MAX_PEERS];
  __shared__ u64 sh_base[MAX_PEERS];
  for (u64 i0 = (u64)blockIdx.x * XT; i0 < n; i0 += (u64)gridDim.x * XT) {
    __syncthreads();
    if (threadIdx.x < MAX_PEERS) sh_count[threadIdx.x] = 0;
    __syncthreads();
    const u64 i = i0 + threadIdx.x;
    u32 dest = 0, rank = 0;
    u64 r[NW];
    if (i < n) {
      load_row<NW>(rows, i, r);
      dest = (u32)(fnv1a64(r[0]) % peers);
      rank = atomicAdd(&sh_count[dest], 1u);
    }
    __syncthreads();
    if (threadIdx.x < peers && sh_count[threadIdx.x])
      sh_base[threadIdx.x] = atomicAdd(&cursors[threadIdx.x], (unsigned long long)sh_count[threadIdx.x]);
    __syncthreads();
    if (i < n) store_row<NW>(out, sh_base[dest] + rank, r);
  }
}

// counts[0..P) -> cursors[0..P) = exclusive offsets (counts stay for the count exchange)
__global__ void k_part_offsets(const unsigned long long* __restrict__ counts, u32 peers,
                               unsigned long long* __restrict__ cursors) {
  if (threadIdx.x == 0) {
    unsigned long long off = 0;
    for (u32 p = 0; p < peers; ++p) {
      cursors[p] = off;
      off += counts[p];
    }
  }
}

// ---- several buffers in one launch (blockIdx.y = buffer): the exchange points of one round
struct PartJobs {
  const u64* rows[MZ_MAX_EXCHANGE];
  u64* out[MZ_MAX_EXCHANGE];
  DLen n[MZ_MAX_EXCHANGE];
  int nw[MZ_MAX_EXCHANGE];
};
__global__ void __launch_bounds__(XT) k_part_count_many(const __grid_constant__ PartJobs jobs, u32 peers,
                                                        unsigned long long* __restrict__ counts /* [job][64] */) {
  const int j = blockIdx.y;
  const u64 n = dlen_get(jobs.n[j]);
  const u64* rows = jobs.rows[j];
  const int nw = jobs.nw[j];
  __shared__ u32 sh[MAX_PEERS];
  if (threadIdx.x < MAX_PEERS) sh[threadIdx.x] = 0;
  __syncthreads();
  for (u64 i = (u64)blockIdx.x * XT + threadIdx.x; i < n; i += (u64)gridDim.x * XT)
    atomicAdd(&sh[(u32)(fnv1a64(rows[i * nw]) % peers)], 1u);
  __syncthreads();
  if (threadIdx.x < peers && sh[threadIdx.x])
    atomicAdd(&counts[j * 64 + threadIdx.x], (unsigned long long)sh[threadIdx.x]);
}
__global__ void k_part_offsets_many(const unsigned long long* __restrict__ counts, u32 peers, u32 k,
                                    unsigned long long* __restrict__ cursors,
                                    unsigned long long* __restrict__ send_by_peer /* [peer][k] */) {
  const u32 j = threadIdx.x;
  if (j < k) {
    unsigned long long off = 0;
    for (u32 p = 0; p < peers; ++p) {
      const unsigned long long cnt = counts[j * 64 + p];
      cursors[j * 64 + p] = off;
      send_by_peer[(size_t)p * k + j] = cnt;  // one message per peer carries all k counts
      off += cnt;
    }
  }
}
__global__ void __launch_bounds__(XT) k_part_scatter_many(const __grid_constant__ PartJobs jobs, u32 peers,
                                                          unsigned long long* __restrict__ cursors) {
  const int j = blockIdx.y;
  const u64 n = dlen_get(jobs.n[j]);
  const u64* rows = jobs.rows[j];
  u64* out = jobs.out[j];
  const int nw = jobs.nw[j];
  __shared__ u32 sh_count[MAX_PEERS];
  __shared__ u64 sh_base[MAX_PEERS];
  for (u64 i0 = (u64)blockIdx.x * XT; i0 < n; i0 += (u64)gridDim.x * XT) {
    __syncthreads();
    if (threadIdx.x < MAX_PEERS) sh_count[threadIdx.x] = 0;
    __syncthreads();
    const u64 i = i0 + threadIdx.x;
    u32 dest = 0, rank = 0;
    if (i < n) {
      dest = (u32)(fnv1a64(rows[i * nw]) % peers);
      rank = atomicAdd(&sh_count[dest], 1u);
    }
    __syncthreads();
    if (threadIdx.x < peers && sh_count[threadIdx.x])
      sh_base[threadIdx.x] = atomicAdd(&cursors[j * 64 + threadIdx.x], (unsigned long long)sh_count[threadIdx.x]);
    __syncthreads();
    if (i < n) {
      const u64* src = rows + i * nw;
      u64* dst = out + (sh_base[dest] + rank) * nw;
      for (int w = 0; w < nw; w += 2) {  // rows are 16-byte multiples (nw even: 4 or 10)
        const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(src + w);
        *reinterpret_cast<ulonglong2*>(dst + w) = v;
      }
    }
  }
}


// =============================================================== exchange over peer memory
// The Exchange pact as ONE scatter kernel that partitions AND delivers: every row is written
// straight into the destination worker's landing zone (NVLink peer stores, or a local store for
// the worker's own share); no NCCL call, no counts all-to-all, no host wait.  A landing zone
// has a fixed-capacity region per (round parity, buffer slot, source worker), so a source
// needs no offsets from anybody: it fills its region from 0 and publishes the count and a
// round flag when its last CTA is done.  The receiving worker's gather kernel waits for the
// flags of all sources (device-side spin on its own memory), then compacts the P regions of
// each slot into the operator's input buffer and leaves the row count on the device.
//
// Region reuse is safe with two parities and no acknowledgements: a worker's stream runs
// scatter(r), gather(r), ..., scatter(r+1), gather(r+1); scatter(r+2) on worker A (same parity
// as r) is ordered after A's gather(r+1), which waited for B's scatter(r+1), which B's stream
// ordered after B's gather(r) -- so B has consumed round r before A overwrites it.

struct P2PJobs {
  const u64* rows[MZ_MAX_EXCHANGE];
  DLen n[MZ_MAX_EXCHANGE];
  int nw[MZ_MAX_EXCHANGE];
  u64* out[MZ_MAX_EXCHANGE];      // gather: destination buffers
  u64 out_cap[MZ_MAX_EXCHANGE];   // gather: their capacities (rows)
  u64* out_len[MZ_MAX_EXCHANGE];  // gather: where the row counts go
};
struct P2PView {
  char* peer[MZ_P2P_MAX_PEERS];  // landing zone bases (peer[me] is local memory)
  u64 L;                         // rows per region
  u32 region_rb;                 // bytes reserved per row in a region
  u32 P, me, k;
  u64 round;
};
__host__ __device__ __forceinline__ u64 p2p_region_off(const P2PView& v, u32 par, u32 slot, u32 src) {
  return (u64)MZ_P2P_HEADER_BYTES + ((((u64)par * MZ_MAX_EXCHANGE + slot) * v.P + src) * v.L) * v.region_rb;
}
// header: flags[2][16] then counts[2][MZ_MAX_EXCHANGE][16], all u64
__host__ __device__ __forceinline__ u64 p2p_flag_off(u32 par, u32 src) { return ((u64)par * 16 + src) * 8; }
__host__ __device__ __forceinline__ u64 p2p_count_off(u32 par, u32 slot, u32 src) {
  return 256 + (((u64)par * MZ_MAX_EXCHANGE + slot) * 16 + src) * 8;
}

__global__ void __launch_bounds__(XT) k_p2p_scatter(const __grid_constant__ P2PJobs jobs,
                                                    const __grid_constant__ P2PView v,
                                                    unsigned long long* __restrict__ cursors /* [slot][16] */,
                                                    u32* __restrict__ done, u64* __restrict__ status) {
  const int j = blockIdx.y;
  const u64 n = dlen_get(jobs.n[j]);
  const u64* rows = jobs.rows[j];
  const int nw = jobs.nw[j];
  const u32 par = (u32)(v.round & 1);
  __shared__ u32 sh_count[MZ_P2P_MAX_PEERS];
  __shared__ u64 sh_base[MZ_P2P_MAX_PEERS];
  __shared__ u32 s_last;
  // P2P_IT rows per thread and round: the keys of a round are loaded together, one range per destination is
  // reserved for all of them with a single global atomic, then the rows go out -- the per-round chain (key
  // load, reservation, stores) is paid once per 1024 rows instead of once per 256
  constexpr int P2P_IT = 4;
  for (u64 i0 = (u64)blockIdx.x * XT * P2P_IT; i0 < n; i0 += (u64)gridDim.x * XT * P2P_IT) {
    __syncthreads();
    if (threadIdx.x < MZ_P2P_MAX_PEERS) sh_count[threadIdx.x] = 0;
    __syncthreads();
    u64 key[P2P_IT];
    u32 dest[P2P_IT], rank[P2P_IT];
#pragma unroll
    for (int u = 0; u < P2P_IT; ++u) {
      const u64 i = i0 + (u64)u * XT + threadIdx.x;
      key[u] = i < n ? rows[i * nw] : 0;
    }
#pragma unroll
    for (int u = 0; u < P2P_IT; ++u) {
      const u64 i = i0 + (u64)u * XT + threadIdx.x;
      dest[u] = 0;
      rank[u] = 0;
      if (i < n) {
        dest[u] = (u32)(fnv1a64(key[u]) % v.P);
        rank[u] = atomicAdd(&sh_count[dest[u]], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x < v.P && sh_count[threadIdx.x])
      sh_base[threadIdx.x] = atomicAdd(&cursors[j * 16 + threadIdx.x], (unsigned long long)sh_count[threadIdx.x]);
    __syncthreads();
#pragma unroll
    for (int u = 0; u < P2P_IT; ++u) {
      const u64 i = i0 + (u64)u * XT + threadIdx.x;
      if (i >= n) continue;
      const u64 at = sh_base[dest[u]] + rank[u];
      if (at < v.L) {
        const u64* src = rows + i * nw;
        u64* dst = (u64*)(v.peer[dest[u]] + p2p_region_off(v, par, (u32)j, v.me)) + at * nw;
        for (int w = 0; w < nw; w += 2) {  // rows are 16-byte multiples
          const ulonglong2 x = *reinterpret_cast<const ulonglong2*>(src + w);
          *reinterpret_cast<ulonglong2*>(dst + w) = x;
        }
      } else {
        atomicMax((unsigned long long*)status, (unsigned long long)(at + 1));  // region overflow: reported, nothing wrong is delivered
      }
    }
  }
  // ---- publish: the last CTA of the launch sends counts and the round flag to every peer
  __threadfence_system();  // this CTA's peer stores are visible system-wide before it counts itself done
  __syncthreads();
  if (threadIdx.x == 0) {
    const u32 total = gridDim.x * gridDim.y;
    const u32 prev = atomicAdd(done, 1u);
    s_last = (prev == total - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (s_last == 0u) return;
  __threadfence();  // the other CTAs' cursor updates (acquire side of the done counter)
  for (u32 t = threadIdx.x; t < v.k * v.P; t += XT) {
    const u32 e = t / v.P, d = t % v.P;
    unsigned long long c = *(volatile unsigned long long*)&cursors[e * 16 + d];
    if (c > v.L) c = v.L;
    *(volatile u64*)(v.peer[d] + p2p_count_off(par, e, v.me)) = (u64)c;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < v.P) {
    u64* flag = (u64*)(v.peer[threadIdx.x] + p2p_flag_off(par, v.me));
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(flag), "l"(v.round) : "memory");
  }
  // ready for the next round (stream-ordered behind this launch)
  for (u32 t = threadIdx.x; t < MZ_MAX_EXCHANGE * 16; t += XT) cursors[t] = 0;
  if (threadIdx.x == 0) *done = 0;
}

__global__ void __launch_bounds__(XT) k_p2p_gather(const __grid_constant__ P2PJobs jobs,
                                                   const __grid_constant__ P2PView v, u64* __restrict__ status) {
  const int j = blockIdx.y;
  const u32 par = (u32)(v.round & 1);
  const char* mine = v.peer[v.me];
  __shared__ u64 s_pref[MZ_P2P_MAX_PEERS + 1];
  // every source's flag for this round (sources publish their counts before the flag)
  if (threadIdx.x < v.P) {
    const u64* flag = (const u64*)(mine + p2p_flag_off(par, threadIdx.x));
    u64 f;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(f) : "l"(flag) : "memory");
    } while (f < v.round);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    u64 acc = 0;
    for (u32 s = 0; s < v.P; ++s) {
      s_pref[s] = acc;
      acc += *(volatile const u64*)(mine + p2p_count_off(par, (u32)j, s));
    }
    s_pref[v.P] = acc;
  }
  __syncthreads();
  const int nw = jobs.nw[j];
  u64 total = s_pref[v.P];
  if (total > jobs.out_cap[j]) {
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicMax((unsigned long long*)status, (unsigned long long)total);
    total = jobs.out_cap[j];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *jobs.out_len[j] = total;
  const u32 cpr = (u32)nw / 2;  // 16-byte chunks per row
  const u64 chunks = total * cpr;
  for (u64 c = (u64)blockIdx.x * XT + threadIdx.x; c < chunks; c += (u64)gridDim.x * XT) {
    const u64 row = c / cpr;
    const u32 w = (u32)(c % cpr) * 2;
    u32 s = 0;
    while (s + 1 < v.P && row >= s_pref[s + 1]) ++s;
    const u64* src = (const u64*)(mine + p2p_region_off(v, par, (u32)j, s)) + (row - s_pref[s]) * nw + w;
    const ulonglong2 x = *reinterpret_cast<const ulonglong2*>(src);
    *reinterpret_cast<ulonglong2*>(jobs.out[j] + row * nw + w) = x;
  }
}

}  // namespace

uint32_t mzgpu_route(uint64_t key, uint32_t peers) { return (uint32_t)(fnv1a64(key) % peers); }

// Bucket rows by destination entirely on the device: d_counts[p] = rows for peer
// p, d_out = rows grouped by destination in peer order.  No host round trip.
int32_t mz_partition(mzgpu_ctx* ctx, int row_bytes, const void* d_rows, DLen n, u64 n_ub, u32 peers, void* d_out,
                     u64* d_counts /* MAX_PEERS words */, u64* d_cursors /* MAX_PEERS words */) {
  if (peers > MAX_PEERS) {
    MZ_SET_ERR(ctx, "exchange: %u peers exceed the supported maximum %d", peers, MAX_PEERS);
    return MZGPU_E_UNSUPPORTED;
  }
  MZ_CUDA(ctx, cudaMemsetAsync(d_counts, 0, MAX_PEERS * 8, ctx->stream));
  if (n_ub == 0) return MZGPU_OK;
  const u64* r = (const u64*)d_rows;
  unsigned long long* c = (unsigned long long*)d_counts;
  unsigned long long* cur = (unsigned long long*)d_cursors;
  u64 blocks = (n_ub + XT - 1) / XT;
  unsigned grid = (unsigned)(blocks < (u64)ctx->num_sms * 8 ? blocks : (u64)ctx->num_sms * 8);
  return mz_dispatch<ExchangeWidths>(ctx, row_bytes, "exchange", [&](auto RB) {
    constexpr int NW = RowT<RB>::NW;
    MZ_LAUNCH(ctx, k_part_count<NW>, grid, XT, 0, r, n, peers, c);
    MZ_LAUNCH(ctx, k_part_offsets, 1, 32, 0, c, peers, cur);
    MZ_LAUNCH(ctx, k_part_scatter<NW>, grid, XT, 0, r, n, peers, cur, (u64*)d_out);
    return MZGPU_OK;
  });
}

// All buffers of one exchange round in three launches (count, offsets, scatter).
// d_counts / d_cursors: [k][64] words.
int32_t mz_partition_many(mzgpu_ctx* ctx, u32 k, const int* row_bytes, const void* const* d_rows, const DLen* n,
                          const u64* n_ub, u32 peers, void* const* d_out, u64* d_counts, u64* d_cursors,
                          u64* d_send_by_peer) {
  if (peers > MAX_PEERS || k > MZ_MAX_EXCHANGE) {
    MZ_SET_ERR(ctx, "exchange: %u peers / %u buffers exceed the supported maximum", peers, k);
    return MZGPU_E_UNSUPPORTED;
  }
  MZ_CUDA(ctx, cudaMemsetAsync(d_counts, 0, (size_t)k * 64 * 8, ctx->stream));
  PartJobs jobs;
  memset(&jobs, 0, sizeof(jobs));
  u64 max_ub = 0;
  for (u32 j = 0; j < k; ++j) {
    if (!ExchangeWidths::has(row_bytes[j])) {
      MZ_SET_ERR(ctx, "exchange: unsupported row width %d", row_bytes[j]);
      return MZGPU_E_UNSUPPORTED;
    }
    jobs.rows[j] = (const u64*)d_rows[j];
    jobs.out[j] = (u64*)d_out[j];
    jobs.n[j] = n[j];
    jobs.nw[j] = row_bytes[j] / 8;
    max_ub = n_ub[j] > max_ub ? n_ub[j] : max_ub;
  }
  u64 blocks = (max_ub + XT - 1) / XT;
  const u64 maxb = (u64)ctx->num_sms * 4;
  if (blocks > maxb) blocks = maxb;
  if (blocks == 0) blocks = 1;
  dim3 grid((unsigned)blocks, k);
  unsigned long long* c = (unsigned long long*)d_counts;
  unsigned long long* cur = (unsigned long long*)d_cursors;
  MZ_LAUNCH(ctx, k_part_count_many, grid, XT, 0, jobs, peers, c);
  MZ_LAUNCH(ctx, k_part_offsets_many, 1, 32, 0, c, peers, k, cur, (unsigned long long*)d_send_by_peer);
  MZ_LAUNCH(ctx, k_part_scatter_many, grid, XT, 0, jobs, peers, cur);
  return MZGPU_OK;
}

// ---- exchange over peer memory: host side of the two kernels above
size_t mz_p2p_zone_bytes(u64 landing_rows, u32 region_rb, u32 peers) {
  return (size_t)MZ_P2P_HEADER_BYTES + (size_t)2 * MZ_MAX_EXCHANGE * peers * landing_rows * region_rb;
}
static void p2p_view(mzgpu_ctx* ctx, u32 k, P2PView* v) {
  memset(v, 0, sizeof(*v));
  for (int p = 0; p < ctx->peers; ++p) v->peer[p] = (char*)ctx->p2p_peer[p];
  v->L = ctx->p2p_rows;
  v->region_rb = ctx->p2p_region_rb;
  v->P = (u32)ctx->peers;
  v->me = (u32)ctx->worker;
  v->k = k;
  v->round = ctx->p2p_round;
}
int32_t mz_p2p_send(mzgpu_ctx* ctx, u32 k, const int* row_bytes, const void* const* d_rows, const DLen* n,
                    const u64* n_ub) {
  P2PJobs jobs;
  memset(&jobs, 0, sizeof(jobs));
  u64 max_ub = 0;
  for (u32 j = 0; j < k; ++j) {
    if ((row_bytes[j] != 32 && row_bytes[j] != 80) || (u32)row_bytes[j] > ctx->p2p_region_rb) {
      MZ_SET_ERR(ctx, "exchange_p2p: row width %d does not fit the landing regions (%u bytes per row)", row_bytes[j],
                 ctx->p2p_region_rb);
      return MZGPU_E_UNSUPPORTED;
    }
    jobs.rows[j] = (const u64*)d_rows[j];
    jobs.n[j] = n[j];
    jobs.nw[j] = row_bytes[j] / 8;
    max_ub = n_ub[j] > max_ub ? n_ub[j] : max_ub;
  }
  P2PView v;
  p2p_view(ctx, k, &v);
  // few, fat CTAs: every CTA ends with a system-wide fence (its peer stores must have landed
  // before it counts itself done), and the last one waits for all of them
  u64 blocks = (max_ub + 4 * XT - 1) / (4 * XT);
  const u64 maxb = std::max<u64>(1, (u64)ctx->num_sms / k);
  if (blocks > maxb) blocks = maxb;
  if (blocks == 0) blocks = 1;
  MZ_LAUNCH(ctx, k_p2p_scatter, dim3((unsigned)blocks, k), XT, 0, jobs, v, (unsigned long long*)ctx->p2p_cursors,
            ctx->p2p_done, ctx->d_status);
  return MZGPU_OK;
}
int32_t mz_p2p_recv(mzgpu_ctx* ctx, u32 k, const int* row_bytes, void* const* d_out, const u64* out_cap,
                    u64* const* d_out_len) {
  P2PJobs jobs;
  memset(&jobs, 0, sizeof(jobs));
  u64 max_cap = 0;
  for (u32 j = 0; j < k; ++j) {
    jobs.nw[j] = row_bytes[j] / 8;
    jobs.out[j] = (u64*)d_out[j];
    jobs.out_cap[j] = out_cap[j];
    jobs.out_len[j] = d_out_len[j];
    max_cap = out_cap[j] > max_cap ? out_cap[j] : max_cap;
  }
  P2PView v;
  p2p_view(ctx, k, &v);
  // few CTAs: they spin until every peer has delivered, and must leave room for whatever else runs
  u64 blocks = (max_cap * 2 + XT - 1) / XT;
  const u64 maxb = (u64)ctx->num_sms;
  if (blocks > maxb) blocks = maxb;
  if (blocks == 0) blocks = 1;
  MZ_LAUNCH(ctx, k_p2p_gather, dim3((unsigned)blocks, k), XT, 0, jobs, v, ctx->d_status);
  return MZGPU_OK;
}
