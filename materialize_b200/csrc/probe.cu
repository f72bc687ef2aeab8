// probe.cu — arrangement probes for the joins (SURVEY.md a8-a10).
//
// Reference:
//   half_join   differential-dogs3 0.23.0 half_join2::half_join_internal_unsafe
//               (external) as configured by build_halfjoin2,
//               src/compute/src/render/join/delta_join.rs:379-484; tie-break
//               comparison `le`/`lt` :204-224; semantics SURVEY.md A8
//   join_core   Work::start_work key merge + Joiner::join_key_simple,
//               src/compute/src/render/join/mz_join_core.rs:591-623,714-726
//               (the pairwise form; the linear time scan :729-793 yields the
//               same consolidated output, SURVEY.md A7)
//
// The CPU operators sort the probe side and walk a merged cursor with
// `seek_key`.  Here every probe row is one thread: a 128-bit load of the hash
// slot per batch of the trace, then a contiguous run of 32-byte lookup rows.
// Two passes (count -> scan -> write) give each probe row a private, bounded
// output range, so the expansion needs no atomics and no output sort.
#include "common.cuh"

namespace {

constexpr int PT = 256;

// visit every (val2, time2, diff2) of `key` in the trace that passes the time
// filter; F(v2, t2, d2)
// `count_runs` != nullptr: the caller only counts, and every row of a run matches (no time
// filter, no closure) -- a run whose length is in the slot adds it without touching the rows.
template <int GROUP, class F>
__device__ __forceinline__ void for_each_match(const TraceView& tv, u64 key, u64 t1, int mode, F f,
                                               u32* count_runs = nullptr) {
  const u64 h0 = mix64(key);
  // The first slot of several batches is fetched before any of them is looked at:
  // the loads are independent, so a probe against a trace of many batches costs
  // about one memory latency per group instead of one per batch (update-batch probes
  // take eight batches per group).
  for (u32 b0 = 0; b0 < tv.n_batches; b0 += GROUP) {
    ulonglong2 slot[GROUP];
    u64 hh[GROUP], mask[GROUP];
#pragma unroll
    for (int j = 0; j < GROUP; ++j) {
      if (b0 + j < tv.n_batches) {
        const BatchView& bv = tv.b[b0 + j];
        mask[j] = bv_mask(bv);
        hh[j] = h0 & mask[j];
        slot[j] = *reinterpret_cast<const ulonglong2*>(&bv.table[hh[j]]);
      }
    }
#pragma unroll
    for (int j = 0; j < GROUP; ++j) {
      if (b0 + j >= tv.n_batches) break;
      const BatchView& bv = tv.b[b0 + j];
      ulonglong2 sl = slot[j];
      u64 h = hh[j];
      while (true) {
        if (sl.y == 0) break;
        if (sl.x == key) {
          const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
          const u32 len = (u32)(sl.y >> 44);
          if (len != 0 && count_runs != nullptr) {
            *count_runs += len;
          } else if (len != 0) {
            // run length known: the rows' loads do not depend on each other
            for (u32 r0 = 0; r0 < len; r0 += 4) {
              ulonglong2 kv[4], td[4];
#pragma unroll
              for (int q = 0; q < 4; ++q)
                if (r0 + q < len) {
                  kv[q] = *reinterpret_cast<const ulonglong2*>(bv.rows + (first + r0 + q) * 4);
                  td[q] = *reinterpret_cast<const ulonglong2*>(bv.rows + (first + r0 + q) * 4 + 2);
                }
#pragma unroll
              for (int q = 0; q < 4; ++q)
                if (r0 + q < len) {
                  bool ok = mode == MZ_PROBE_HALF_LE ? td[q].x <= t1 : (mode == MZ_PROBE_HALF_LT ? td[q].x < t1 : true);
                  if (ok) f(kv[q].y, td[q].x, (i64)td[q].y);
                }
            }
          } else {
            const u64 bn = bv_n(bv);
            for (u64 r = first; r < bn; ++r) {
              const ulonglong2 kv = *reinterpret_cast<const ulonglong2*>(bv.rows + r * 4);
              if (kv.x != key) break;
              const ulonglong2 td = *reinterpret_cast<const ulonglong2*>(bv.rows + r * 4 + 2);
              bool ok = mode == MZ_PROBE_HALF_LE ? td.x <= t1 : (mode == MZ_PROBE_HALF_LT ? td.x < t1 : true);
              if (ok) f(kv.y, td.x, (i64)td.y);
            }
          }
          break;
        }
        h = (h + 1) & mask[j];
        sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      }
    }
  }
}

// ---- single-pass forms: sizes come from device memory, results are appended at
// a device-resident offset, the new length is left in device memory.  Tiles are
// chained with a decoupled look-back, so the output order is exactly the
// two-pass order (stream order x batch order x row order) and nothing returns
// to the host.
//
// A tile is expanded by the whole CTA.  The reference's half_join walks a cursor per key; a
// thread per probe row doing the same serialises on memory latency (a key with rows in three
// batches = a dozen dependent DRAM round trips, and the rest of the CTA waits at the scan
// barrier).  Here:
//   1. thread per probe row: first slot of every batch (independent loads), hits counted;
//   2. block scans give every hit its place in the tile's hit list (thread-major, batch order)
//      and the tile's CANDIDATE list (the rows of every hit run, concatenated);
//   3. the candidates are split evenly over the warps: each lane loads one lookup row per step
//      (independent loads, any fan-out, any skew inside the tile), applies the time filter and
//      the closure, and counts the survivors; look-back; the same walk again writes them
//      (rows come from L1/L2 the second time) at offsets from warp ballots -- no block barrier
//      inside either walk.
// Rows per tile shrink with the number of batches so that the hit list always fits
// (hits <= rows x batches <= PROBE_HCAP).
constexpr int PROBE_WHCAP = 256;  // hits one WARP's share of a tile can hold (rows x batches)
struct ProbeWarpSmem {
  u32 hit_pref[PROBE_WHCAP + 1];  // candidates before hit h (exclusive); [n_hits] = all candidates
  u64 hit_first[PROBE_WHCAP];     // first row of the run | batch index << 48
  uint8_t hit_lane[PROBE_WHCAP];  // lane that owns the probe row
};
struct ProbeSmem {
  u32 tile;
  u64 bcast;
  u32 warp_keep[PT / 32];
  ProbeWarpSmem w[PT / 32];
};

// The closure a probe applies to each match: the bit-field closure of ProbeParams (mzgpu_closure, or the R40
// identity without one), or an MfpPlan (mzgpu_join_closure) over the words (key, va, vb) whose errors become R32
// rows (code, payload, time, diff) at warp-aggregated slots *err_len++ of `errs` (err_cap rows; the host sizes it
// so that it cannot fill, a slot past it is reported through the status word and not written).
struct BitClosure {
  static constexpr bool MFP = false;
};
struct MfpClosure {
  static constexpr bool MFP = true;
  const MfpDevPlan* pl;
  u64* errs;
  u64 err_cap;
  unsigned long long* err_len;
};

struct ProbePre {  // optional map in front of the probe (build_update_stream fused in)
  int has_pre, pre_has_closure;
  u64 skip_time;
  const mzgpu_closure* pre;
};

// first matching slot of `key` in batch `bv`: {first row, run length} or len = 0 when absent
__device__ __forceinline__ bool probe_slot_resolve(const BatchView& bv, u64 key, ulonglong2 sl, u64 h, u64 mask,
                                                   u64* first, u32* len) {
  // linear probing: after the first slot, FOUR slots per round trip (independent loads, mostly one
  // 64-byte sector).  A tile resolves a couple of thousand slots and waits for the longest chain
  // among them (~10 steps at load factor 0.5): one memory latency per step was the tile's tail.
  while (sl.y != 0 && sl.x != key) {
    ulonglong2 q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) q[i] = *reinterpret_cast<const ulonglong2*>(&bv.table[(h + 1 + i) & mask]);
    bool settled = false;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (!settled && (q[i].y == 0 || q[i].x == key)) {
        sl = q[i];
        settled = true;
      }
    if (settled) break;
    h = (h + 4) & mask;
    sl = q[3];  // occupied by another key: the loop goes on from the slot after it
  }
  if (sl.y == 0) return false;
  const u64 f = (sl.y & MZ_SLOT_ROW_MASK) - 1;
  u32 l = (u32)(sl.y >> 44);
  if (l == 0) {
    // the builder did not record the run length (a long run): rows are sorted by key, so the end
    // of the run is an upper-bound search
    u64 lo = f + 1, hi = bv_n(bv);
    while (lo < hi) {
      const u64 mid = (lo + hi) >> 1;
      if (bv.rows[mid * 4] == key)
        lo = mid + 1;
      else
        hi = mid;
    }
    const u64 run = lo - f;
    l = run > 0xffffffffull ? 0xffffffffu : (u32)run;
  }
  *first = f;
  *len = l;
  return true;
}

__device__ __forceinline__ u32 warp_exclusive_scan(u32 v, u32* total) {
  const u32 lane = threadIdx.x & 31;
  u32 incl = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const u32 o = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= (u32)off) incl += o;
  }
  *total = __shfl_sync(0xffffffffu, incl, 31);
  return incl - v;
}

// One tile: probe rows [row0, row0 + 8 * TRW) of `stream` (n rows) against `tv`: warp w takes rows
// [row0 + w * TRW, + TRW), one per lane.  The warps of the CTA run on their own -- private hit
// lists, warp scans, no block barrier -- up to the point where the tile's total is needed for the
// look-back (one barrier), so one warp's memory latency never stalls the other seven.
template <int OUT_NW, class CL>
__device__ __forceinline__ void probe_tile(ProbeSmem& S, const u64* __restrict__ stream, u64 n, u64 row0, u32 TRW,
                                           const TraceView& tv, const ProbeParams& pp, const ProbePre& pre,
                                           const LookBack& lb, u32 tile, u64* __restrict__ out, u64 base0,
                                           u64 out_cap, u64* __restrict__ status, u64* excl_out, u32* total_out,
                                           const CL& cl) {
  constexpr int GROUP = 8;
  // candidates per lane and step: their searches and row loads overlap (an MfpPlan closure keeps one: the
  // interpreter's state leaves no registers for more)
  constexpr int U = CL::MFP ? 1 : 4;
  const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ProbeWarpSmem& W = S.w[warp];
  // ---- 1. this lane's probe row
  const u64 i = row0 + (u64)warp * TRW + lane;
  u64 key = 0, v1 = 0, t1 = 0, d1 = 0;
  bool live = lane < TRW && i < n;
  if (live) {
    const ulonglong2 kv = *reinterpret_cast<const ulonglong2*>(stream + i * 4);
    const ulonglong2 td = *reinterpret_cast<const ulonglong2*>(stream + i * 4 + 2);
    key = kv.x;
    v1 = kv.y;
    t1 = td.x;
    d1 = td.y;
    if (pre.has_pre) {
      if (pre.skip_time != MZGPU_FRONTIER_EMPTY && t1 == pre.skip_time) {
        live = false;
      } else if (pre.pre_has_closure) {
        u64 k, v;
        if (closure_eval(*pre.pre, key, v1, 0, &k, &v)) {
          key = k;
          v1 = v;
        } else {
          live = false;
        }
      }
    }
  }
  const u64 h0 = mix64(key);
  // ---- 2. hits: first slot of every batch (independent loads), warp scans, private hit list.
  // A trace of at most GROUP batches keeps its hits in registers (one walk of the slots); a
  // longer one walks the slots twice (the second time from L1).
  u32 hit_off = 0, cand_off = 0, n_hits = 0, n_cand = 0;
  const bool one_group = tv.n_batches <= (u32)GROUP;
  u64 reg_first[GROUP];
  u32 reg_len[GROUP];
#pragma unroll
  for (int j = 0; j < GROUP; ++j) reg_len[j] = 0;
#pragma unroll 1
  for (int phase = 0; phase < 2; ++phase) {
    u32 k_hit = 0, k_cand = 0;
    if (phase == 1 && one_group) {
#pragma unroll
      for (int j = 0; j < GROUP; ++j)
        if (reg_len[j] != 0) {
          const u32 h = hit_off + k_hit;
          W.hit_first[h] = reg_first[j] | ((u64)j << 48);
          W.hit_lane[h] = (uint8_t)lane;
          W.hit_pref[h] = cand_off + k_cand;
          k_hit++;
          k_cand += reg_len[j];
        }
    } else if (live) {
#pragma unroll 1
      for (u32 b0 = 0; b0 < tv.n_batches; b0 += GROUP) {
        ulonglong2 slot[GROUP];
        u64 hh[GROUP], msk[GROUP];
#pragma unroll
        for (int j = 0; j < GROUP; ++j) {
          if (b0 + j < tv.n_batches) {
            const BatchView& bv = tv.b[b0 + j];
            msk[j] = bv_mask(bv);
            hh[j] = h0 & msk[j];
            slot[j] = *reinterpret_cast<const ulonglong2*>(&bv.table[hh[j]]);
          }
        }
#pragma unroll
        for (int j = 0; j < GROUP; ++j) {
          if (b0 + j >= tv.n_batches) break;
          u64 first;
          u32 len;
          if (!probe_slot_resolve(tv.b[b0 + j], key, slot[j], hh[j], msk[j], &first, &len)) continue;
          if (phase == 0 && one_group) {
            reg_first[j] = first;
            reg_len[j] = len;
          }
          if (phase == 1) {
            const u32 h = hit_off + k_hit;
            W.hit_first[h] = first | ((u64)(b0 + j) << 48);
            W.hit_lane[h] = (uint8_t)lane;
            W.hit_pref[h] = cand_off + k_cand;
          }
          k_hit++;
          k_cand += len;
        }
      }
    }
    if (phase == 0) {
      hit_off = warp_exclusive_scan(k_hit, &n_hits);
      cand_off = warp_exclusive_scan(k_cand, &n_cand);
    }
  }
  if (lane == 0) W.hit_pref[n_hits] = n_cand;
  __syncwarp();
  // ---- 3. the candidate walk (pass 0 counts, pass 1 writes).  The first 32 * U candidates --
  // all of them for most warps -- are evaluated once and kept in registers across the look-back.
  // An MfpPlan closure's error (*err) leaves its R32 error row in row[0..4); it is written in pass 1 only.
  auto eval = [&](u32 c, bool valid, u64* row, bool* err) -> bool {
    // the hit this candidate belongs to: last h with hit_pref[h] <= c
    u32 lo = 0, hi = n_hits;
    while (hi - lo > 1) {
      const u32 mid = (lo + hi) >> 1;
      if (W.hit_pref[mid] <= c)
        lo = mid;
      else
        hi = mid;
    }
    u32 owner = 0;
    ulonglong2 rkv = make_ulonglong2(0, 0), rtd = make_ulonglong2(0, 0);
    if (valid) {
      const u64 hf = W.hit_first[lo];
      const BatchView& bv = tv.b[(u32)(hf >> 48)];
      const u64 r = (hf & MZ_SLOT_ROW_MASK) + (u64)(c - W.hit_pref[lo]);
      owner = W.hit_lane[lo];
      rkv = *reinterpret_cast<const ulonglong2*>(bv.rows + r * 4);
      rtd = *reinterpret_cast<const ulonglong2*>(bv.rows + r * 4 + 2);
    }
    // the probe row lives in its owner lane's registers
    const u64 pk = __shfl_sync(0xffffffffu, key, owner), pv = __shfl_sync(0xffffffffu, v1, owner);
    const u64 pt = __shfl_sync(0xffffffffu, t1, owner), pd = __shfl_sync(0xffffffffu, d1, owner);
    if (!valid) return false;
    const u64 t2 = rtd.x;
    bool keep = pp.mode == MZ_PROBE_HALF_LE ? t2 <= pt : (pp.mode == MZ_PROBE_HALF_LT ? t2 < pt : true);
    if (!keep) return false;
    u64 t = pt;
    if (pp.mode == MZ_PROBE_JOIN) {
      t = pt > t2 ? pt : t2;
      t = t > pp.meet ? t : pp.meet;
    }
    const u64 d = pd * rtd.y;
    const u64 va = pp.swap_vals ? rkv.y : pv, vb = pp.swap_vals ? pv : rkv.y;
    if constexpr (CL::MFP) {
      const u64 w[3] = {pk, va, vb};
      u64 mv[MZGPU_MFP_MAX_MAPS];
      u32 e_code = 0;
      u64 e_pay = 0;
      keep = mfp_filter_map(*cl.pl, w, mv, &e_code, &e_pay);
      if (e_code) {
        *err = true;
        row[0] = e_code;
        row[1] = e_pay;
        row[2] = t;
        row[3] = d;
        return false;
      }
      if (!keep) return false;
      mfp_project<OUT_NW>(*cl.pl, w, mv, row);
      row[OUT_NW - 2] = t;
      row[OUT_NW - 1] = d;
    } else if (OUT_NW == 4) {
      u64 k, v;
      keep = closure_eval(pp.closure, pk, va, vb, &k, &v);
      row[0] = k;
      row[1] = v;
      row[2] = t;
      row[3] = d;
    } else {
      row[0] = pk;
      row[1] = va;
      row[2] = vb;
      row[3] = t;
      row[OUT_NW - 1] = d;
    }
    return keep;
  };
  bool keep0[U], err0[U];
  u64 row0r[U][OUT_NW];
  u32 run = 0;
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const u32 c = (u32)u * 32 + lane;
    err0[u] = false;
    keep0[u] = eval(c, c < n_cand, row0r[u], &err0[u]);
    run += __popc(__ballot_sync(0xffffffffu, keep0[u]));
  }
#pragma unroll 1
  for (u32 c0 = 32 * U; c0 < n_cand; c0 += 32) {  // (rare: more than 128 candidates in one warp)
    u64 row[OUT_NW];
    bool err = false;
    const bool k = eval(c0 + lane, c0 + lane < n_cand, row, &err);
    run += __popc(__ballot_sync(0xffffffffu, k));
  }
  // ---- 4. the tile's total, the look-back
  if (lane == 0) S.warp_keep[warp] = run;
  __syncthreads();
  u32 mine = 0, total = 0;
#pragma unroll
  for (int w = 0; w < PT / 32; ++w) {
    const u32 v = S.warp_keep[w];
    if ((u32)w < warp) mine += v;
    total += v;
  }
  const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &S.bcast);
  u64 pos = base0 + excl + mine;
  // ---- 5. write
  auto put = [&](bool keep, bool err, const u64* row) {
    if constexpr (CL::MFP) {
      const u64 p = warp_reserve(err ? 1u : 0u, cl.err_len);
      if (err && p >= cl.err_cap) {
        atomicMax((unsigned long long*)status, ~0ull);
      } else if (err) {
        u64* o = cl.errs + p * 4;
#pragma unroll
        for (int w = 0; w < 4; ++w) o[w] = row[w];
      }
    }
    const u32 m = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const u64 p = pos + __popc(m & ((1u << lane) - 1));
      if (p >= out_cap) {
        atomicMax((unsigned long long*)status, (unsigned long long)(p + 1));
      } else {
        u64* o = out + p * OUT_NW;
#pragma unroll
        for (int w = 0; w < OUT_NW; ++w) o[w] = row[w];
      }
    }
    pos += __popc(m);
  };
#pragma unroll
  for (int u = 0; u < U; ++u) put(keep0[u], err0[u], row0r[u]);
#pragma unroll 1
  for (u32 c0 = 32 * U; c0 < n_cand; c0 += 32) {
    u64 row[OUT_NW];
    bool err = false;
    const bool k = eval(c0 + lane, c0 + lane < n_cand, row, &err);
    put(k, err, row);
  }
  *excl_out = excl;
  *total_out = total;
}

template <int OUT_NW, class CL = BitClosure>
__global__ void __launch_bounds__(PT, 3) k_probe_lb(const u64* __restrict__ stream, const DLen dn,
                                                 const __grid_constant__ TraceView tv,
                                                 const __grid_constant__ ProbeParams pp, const LookBack lb,
                                                 u64* __restrict__ out, const DLen out_base, u64 out_cap,
                                                 u64* __restrict__ out_len, u64* __restrict__ status, u32 tile_rows,
                                                 const CL cl) {
  __shared__ ProbeSmem S;
  const u64 n = dlen_get(dn);
  const u32 TR = tile_rows;
  const u64 n_tiles = (n + TR - 1) / TR;
  const u64 base0 = dlen_get(out_base);
  ProbePre pre;
  pre.has_pre = 0;
  pre.pre_has_closure = 0;
  pre.skip_time = MZGPU_FRONTIER_EMPTY;
  pre.pre = nullptr;
  while (true) {
    const u32 tile = lb_next_tile(lb, &S.tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = base0;
      break;
    }
    u64 excl;
    u32 total;
    probe_tile<OUT_NW, CL>(S, stream, n, (u64)tile * TR, TR / (PT / 32), tv, pp, pre, lb, tile, out, base0, out_cap,
                           status, &excl, &total, cl);
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = base0 + excl + total;
  }
}

// ---- several probes in one launch.  A *chain* is a sequence of probe jobs whose results are
// appended, in job order, to ONE output buffer (the last stage of the delta paths: every path
// appends to the result collection); chains are independent of each other (an earlier stage: one
// output buffer per path).  A chain numbers the tiles of its jobs consecutively and runs one
// look-back over all of them, so its output is exactly what its jobs would have appended one
// after the other; blockIdx.y selects the chain.
constexpr int PROBE_MANY_MAX = MZ_PROBE_MANY_MAX;
struct ProbeJobDev {
  const u64* stream;
  DLen dn;
  TraceView tv;
  ProbeParams pp;
  // optional map in front of the probe (build_update_stream fused into the first half join,
  // delta_join.rs:312-377): rows at `skip_time` are dropped, the closure rewrites (key, val) or drops
  int has_pre, pre_has_closure;
  u64 skip_time;
  mzgpu_closure pre;
  u32 tile_rows;  // probe rows per tile (mz_probe_tile_rows)
};
struct ProbeChain {
  u32 first, count;  // jobs [first, first + count)
  LookBack lb;
  u64* out;
  DLen out_base;
  u64 out_cap;
  u64* out_len;
};
struct ProbeMany {
  u32 n_chains;
  u32 ctas[PROBE_MANY_MAX];  // CTAs of the launch that work on chain c (blockIdx.y = c, blockIdx.x < ctas[c])
  ProbeChain chain[PROBE_MANY_MAX];
  ProbeJobDev job[PROBE_MANY_MAX];
};
static_assert(sizeof(ProbeMany) <= 32000, "kernel parameter space");
// the closure policy of each job of a launch (a job's MfpPlan lives in device memory: three more plans would not fit)
template <class CL>
struct ProbeClosures {
  CL c[PROBE_MANY_MAX];
};

template <int OUT_NW, class CL = BitClosure>
__global__ void __launch_bounds__(PT, 3) k_probe_chains(const __grid_constant__ ProbeMany m,
                                                     u64* __restrict__ status,
                                                     const __grid_constant__ ProbeClosures<CL> cls) {
  __shared__ ProbeSmem S;
  // The chains of a launch differ in size by an order of magnitude (the lineitem path of a Q3 step
  // carries four times the rows of the orders path, the customer path none): the resident CTAs are
  // shared out in proportion to the chains' tile counts (host bounds), not equally -- an equal split
  // leaves the longest chain running four tiles deep on a third of the machine.  A chain's tiles are handed out by ticket to whichever of
  // its CTAs is free, so the look-back never waits for a CTA that has not started.
  if (blockIdx.x >= m.ctas[blockIdx.y]) return;
  const ProbeChain& ch = m.chain[blockIdx.y];
  u64 nj[PROBE_MANY_MAX], tiles_before[PROBE_MANY_MAX + 1];
  u32 trj[PROBE_MANY_MAX];
  tiles_before[0] = 0;
#pragma unroll
  for (int q = 0; q < PROBE_MANY_MAX; ++q) {
    nj[q] = (u32)q < ch.count ? dlen_get(m.job[ch.first + q].dn) : 0;
    trj[q] = (u32)q < ch.count ? m.job[ch.first + q].tile_rows : 256u;
    tiles_before[q + 1] = tiles_before[q] + (nj[q] + trj[q] - 1) / trj[q];
  }
  const u64 n_tiles = tiles_before[PROBE_MANY_MAX];
  const u64 base0 = dlen_get(ch.out_base);
  while (true) {
    const u32 tile = lb_next_tile(ch.lb, &S.tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *ch.out_len = base0;
      break;
    }
    u32 q = 0;
    while (q + 1 < ch.count && (u64)tile >= tiles_before[q + 1]) ++q;
    const ProbeJobDev& J = m.job[ch.first + q];
    ProbePre pre;
    pre.has_pre = J.has_pre;
    pre.pre_has_closure = J.pre_has_closure;
    pre.skip_time = J.skip_time;
    pre.pre = &J.pre;
    u64 excl;
    u32 total;
    probe_tile<OUT_NW, CL>(S, J.stream, nj[q], (u64)(tile - tiles_before[q]) * trj[q], trj[q] / (PT / 32), J.tv, J.pp,
                           pre, ch.lb, tile, ch.out, base0, ch.out_cap, status, &excl, &total, cls.c[ch.first + q]);
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *ch.out_len = base0 + excl + total;
  }
}

__global__ void __launch_bounds__(PT) k_map_rows_lb(const u64* __restrict__ rows, const DLen dn,
                                                    const __grid_constant__ mzgpu_closure cl, int has_closure,
                                                    u64 skip_time, const LookBack lb, u64* __restrict__ out,
                                                    const DLen out_base, u64 out_cap, u64* __restrict__ out_len,
                                                    u64* __restrict__ status) {
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  const u64 n = dlen_get(dn);
  const u64 n_tiles = (n + PT - 1) / PT;
  const u64 base0 = dlen_get(out_base);
  while (true) {
    const u32 tile = lb_next_tile(lb, &s_tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = base0;
      break;
    }
    const u64 i = (u64)tile * PT + threadIdx.x;
    u32 keep = 0;
    u64 r[4] = {0, 0, 0, 0};
    if (i < n) {
      load_row<4>(rows, i, r);
      keep = 1;
      if (skip_time != MZGPU_FRONTIER_EMPTY && r[2] == skip_time) keep = 0;
      if (keep && has_closure) {
        u64 k, v;
        if (closure_eval(cl, r[0], r[1], 0, &k, &v)) {
          r[0] = k;
          r[1] = v;
        } else {
          keep = 0;
        }
      }
    }
    u32 total;
    const u32 ex = block_exclusive_scan(keep, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &s_b);
    if (keep) {
      const u64 pos = base0 + excl + ex;
      if (pos >= out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + 1));
      else
        store_row<4>(out, pos, r);
    }
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = base0 + excl + total;
  }
}

// An MfpPlan closure (CL::MFP): the count pass counts the output rows per probe row and adds the error rows to
// *cl.err_len; the write pass writes both, the errors at slots *cl.err_len++ (a second counter).
template <int OUT_NW, bool WRITE, class CL = BitClosure>
__global__ void __launch_bounds__(PT) k_probe(const u64* __restrict__ stream, u64 n,
                                              const __grid_constant__ TraceView tv,
                                              const __grid_constant__ ProbeParams pp,
                                              u32* __restrict__ tile_counts,
                                              const u32* __restrict__ tile_base,
                                              u32* __restrict__ row_counts,
                                              u64* __restrict__ out, const CL cl) {
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * PT + threadIdx.x;
  u64 key = 0, v1 = 0, t1 = 0;
  i64 d1 = 0;
  u32 cnt = 0;
  if (i < n) {
    if (!WRITE) {
      // the count pass needs the key and the time only
      key = stream[i * 4];
      t1 = stream[i * 4 + 2];
      v1 = pp.has_closure ? stream[i * 4 + 1] : 0;
      if constexpr (CL::MFP) {
        v1 = stream[i * 4 + 1];
        u32 errs = 0;
        for_each_match<1>(tv, key, t1, pp.mode, [&](u64 v2, u64 t2, i64 d2) {
          const u64 w[3] = {key, pp.swap_vals ? v2 : v1, pp.swap_vals ? v1 : v2};
          u64 mv[MZGPU_MFP_MAX_MAPS];
          u32 e_code = 0;
          u64 e_pay = 0;
          if (mfp_filter_map(*cl.pl, w, mv, &e_code, &e_pay)) cnt++;
          if (e_code) errs++;
        });
        if (errs) atomicAdd(cl.err_len, (unsigned long long)errs);
        row_counts[i] = cnt;
      }
      u32 runs = 0;
      const bool whole_runs = pp.mode == MZ_PROBE_JOIN && !pp.has_closure;
      if constexpr (!CL::MFP) for_each_match<1>(
          tv, key, t1, pp.mode,
          [&](u64 v2, u64 t2, i64 d2) {
            if (pp.has_closure) {
              u64 k, v;
              if (closure_eval(pp.closure, key, pp.swap_vals ? v2 : v1, pp.swap_vals ? v1 : v2, &k, &v)) cnt++;
            } else {
              cnt++;
            }
          },
          whole_runs ? &runs : nullptr);
      cnt += runs;
      if constexpr (!CL::MFP) row_counts[i] = cnt;
    } else {
      // the write pass takes the row's count from the count pass: one walk per pass
      cnt = row_counts[i];
      const ulonglong2 kv = *reinterpret_cast<const ulonglong2*>(stream + i * 4);
      const ulonglong2 td = *reinterpret_cast<const ulonglong2*>(stream + i * 4 + 2);
      key = kv.x;
      v1 = kv.y;
      t1 = td.x;
      d1 = (i64)td.y;
    }
  }
  u32 total;
  u32 ex = block_exclusive_scan(cnt, sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
    return;
  }
  if (i < n && (cnt > 0 || CL::MFP)) {
    u64 pos = (u64)tile_base[blockIdx.x] + ex;
    for_each_match<1>(tv, key, t1, pp.mode, [&](u64 v2, u64 t2, i64 d2) {
      u64 t = t1;
      if (pp.mode == MZ_PROBE_JOIN) {
        t = t1 > t2 ? t1 : t2;
        t = t > pp.meet ? t : pp.meet;
      }
      u64 d = (u64)d1 * (u64)d2;
      u64 a = pp.swap_vals ? v2 : v1, b = pp.swap_vals ? v1 : v2;
      if constexpr (CL::MFP) {
        const u64 w[3] = {key, a, b};
        u64 mv[MZGPU_MFP_MAX_MAPS];
        u32 e_code = 0;
        u64 e_pay = 0;
        if (mfp_filter_map(*cl.pl, w, mv, &e_code, &e_pay)) {
          u64 r[OUT_NW];
          mfp_project<OUT_NW>(*cl.pl, w, mv, r);
          r[OUT_NW - 2] = t;
          r[OUT_NW - 1] = d;
          store_row<OUT_NW>(out, pos, r);
          pos++;
        } else if (e_code) {
          const u64 p = atomicAdd(cl.err_len, 1ull);
          if (p < cl.err_cap) {
            u64 e[4] = {e_code, e_pay, t, d};
            store_row<4>(cl.errs, p, e);
          }
        }
      } else if (OUT_NW == 4) {
        u64 k, v;
        if (closure_eval(pp.closure, key, a, b, &k, &v)) {
          u64 r[4] = {k, v, t, d};
          store_row<4>(out, pos, r);
          pos++;
        }
      } else {
        u64* o = out + pos * 5;
        o[0] = key;
        o[1] = a;
        o[2] = b;
        o[3] = t;
        o[4] = d;
        pos++;
      }
    });
  }
}

// closure over R32 rows (val2 = 0), optional skip of one time
template <bool WRITE>
__global__ void __launch_bounds__(PT) k_map_rows(const u64* __restrict__ rows, u64 n,
                                                 const __grid_constant__ mzgpu_closure cl, int has_closure,
                                                 u64 skip_time, u32* __restrict__ tile_counts,
                                                 const u32* __restrict__ tile_base,
                                                 u64* __restrict__ out) {
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * PT + threadIdx.x;
  u32 keep = 0;
  u64 r[4] = {0, 0, 0, 0};
  if (i < n) {
    load_row<4>(rows, i, r);
    keep = 1;
    if (skip_time != MZGPU_FRONTIER_EMPTY && r[2] == skip_time) keep = 0;
    if (keep && has_closure) {
      u64 k, v;
      if (closure_eval(cl, r[0], r[1], 0, &k, &v)) {
        r[0] = k;
        r[1] = v;
      } else {
        keep = 0;
      }
    }
  }
  u32 total;
  u32 ex = block_exclusive_scan(keep, sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
    return;
  }
  if (keep) store_row<4>(out, (u64)tile_base[blockIdx.x] + ex, r);
}

MfpClosure mfp_closure(const MfpProbe& m, u64* errs, u64 err_cap, u64* err_len) {
  MfpClosure c;
  c.pl = m.pl;
  c.errs = errs;
  c.err_cap = err_cap;
  c.err_len = (unsigned long long*)err_len;
  return c;
}

}  // namespace

static int32_t mz_probe_mfp(mzgpu_ctx* ctx, const u64* d_stream, u64 n, const TraceView& trace, const ProbeParams& pp,
                            const MfpProbe& mfp, DevMem* out, u64* n_out, DevMem* errs, u64* n_errs);

int32_t mz_probe(mzgpu_ctx* ctx, const u64* d_stream, u64 n, const TraceView& trace,
                 const ProbeParams& pp, DevMem* out, u64* n_out, const MfpProbe* mfp, DevMem* errs, u64* n_errs) {
  *n_out = 0;
  if (mfp != nullptr) return mz_probe_mfp(ctx, d_stream, n, trace, pp, *mfp, out, n_out, errs, n_errs);
  const int out_rb = pp.has_closure ? 32 : 40;
  if (n == 0 || trace.n_batches == 0) return out->alloc(ctx, 16);
  const u64 n_tiles = (n + PT - 1) / PT;
  DevMem tiles, row_counts;
  MZ_TRY(tiles.alloc(ctx, n_tiles * 4));
  MZ_TRY(row_counts.alloc(ctx, n * 4));
  u64* d_total = ctx->d_scratch + 28;
  if (pp.has_closure) {
    MZ_LAUNCH(ctx, (k_probe<4, false>), (unsigned)n_tiles, PT, 0, d_stream, n, trace, pp, tiles.as<u32>(),
              (const u32*)nullptr, row_counts.as<u32>(), (u64*)nullptr, BitClosure{});
  } else {
    MZ_LAUNCH(ctx, (k_probe<5, false>), (unsigned)n_tiles, PT, 0, d_stream, n, trace, pp, tiles.as<u32>(),
              (const u32*)nullptr, row_counts.as<u32>(), (u64*)nullptr, BitClosure{});
  }
  MZ_LAUNCH(ctx, k_scan_tiles, 1, 1024, 0, tiles.as<u32>(), n_tiles, d_total);
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 28, d_total, 8, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 8;
  const u64 total = ctx->h_scratch[28];
  MZ_TRY(out->alloc(ctx, total * out_rb));
  *n_out = total;
  if (total == 0) return MZGPU_OK;
  // probe row 32 B + one 16 B slot per batch + 32 B per matched row + output row
  MZ_BYTES(ctx, n * (32 + 16 * trace.n_batches) + total * (32 + out_rb));
  if (pp.has_closure) {
    MZ_LAUNCH(ctx, (k_probe<4, true>), (unsigned)n_tiles, PT, 0, d_stream, n, trace, pp, (u32*)nullptr,
              tiles.as<u32>(), row_counts.as<u32>(), out->as<u64>(), BitClosure{});
  } else {
    MZ_LAUNCH(ctx, (k_probe<5, true>), (unsigned)n_tiles, PT, 0, d_stream, n, trace, pp, (u32*)nullptr,
              tiles.as<u32>(), row_counts.as<u32>(), out->as<u64>(), BitClosure{});
  }
  return MZGPU_OK;
}

// The two-pass probe with an MfpPlan closure: the count pass counts output rows per probe row and the error rows
// in all (one wait reads both totals), the write pass writes the output rows in order and the error rows at
// atomic slots of an exactly sized array.
static int32_t mz_probe_mfp(mzgpu_ctx* ctx, const u64* d_stream, u64 n, const TraceView& trace, const ProbeParams& pp,
                            const MfpProbe& mfp, DevMem* out, u64* n_out, DevMem* errs, u64* n_errs) {
  *n_errs = 0;
  if (n == 0 || trace.n_batches == 0) {
    MZ_TRY(errs->alloc(ctx, 16));
    return out->alloc(ctx, 16);
  }
  const u64 n_tiles = (n + PT - 1) / PT;
  DevMem tiles, row_counts;
  MZ_TRY(tiles.alloc(ctx, n_tiles * 4));
  MZ_TRY(row_counts.alloc(ctx, n * 4));
  u64* d_total = ctx->d_scratch + 28;  // [0] output rows (k_scan_tiles), [1] error rows
  u64* d_errs = ctx->d_scratch + 29;
  MZ_CUDA(ctx, cudaMemsetAsync(d_errs, 0, 8, ctx->stream));
  const MfpClosure cnt = mfp_closure(mfp, nullptr, 0, d_errs);
  if (mfp.out_rb == 32) {
    MZ_LAUNCH(ctx, (k_probe<4, false, MfpClosure>), (unsigned)n_tiles, PT, 0, d_stream, n, trace, pp, tiles.as<u32>(),
              (const u32*)nullptr, row_counts.as<u32>(), (u64*)nullptr, cnt);
  } else {
    MZ_LAUNCH(ctx, (k_probe<5, false, MfpClosure>), (unsigned)n_tiles, PT, 0, d_stream, n, trace, pp, tiles.as<u32>(),
              (const u32*)nullptr, row_counts.as<u32>(), (u64*)nullptr, cnt);
  }
  MZ_LAUNCH(ctx, k_scan_tiles, 1, 1024, 0, tiles.as<u32>(), n_tiles, d_total);
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 28, d_total, 16, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 16;
  const u64 total = ctx->h_scratch[28], n_err = ctx->h_scratch[29];
  MZ_TRY(out->alloc(ctx, total * mfp.out_rb));
  MZ_TRY(errs->alloc(ctx, n_err * 32));
  *n_out = total;
  *n_errs = n_err;
  if (total == 0 && n_err == 0) return MZGPU_OK;
  MZ_BYTES(ctx, n * (32 + 16 * trace.n_batches) + total * (32 + mfp.out_rb) + n_err * 64);
  MZ_CUDA(ctx, cudaMemsetAsync(d_errs, 0, 8, ctx->stream));
  const MfpClosure wr = mfp_closure(mfp, errs->as<u64>(), n_err, d_errs);
  if (mfp.out_rb == 32) {
    MZ_LAUNCH(ctx, (k_probe<4, true, MfpClosure>), (unsigned)n_tiles, PT, 0, d_stream, n, trace, pp, (u32*)nullptr,
              tiles.as<u32>(), row_counts.as<u32>(), out->as<u64>(), wr);
  } else {
    MZ_LAUNCH(ctx, (k_probe<5, true, MfpClosure>), (unsigned)n_tiles, PT, 0, d_stream, n, trace, pp, (u32*)nullptr,
              tiles.as<u32>(), row_counts.as<u32>(), out->as<u64>(), wr);
  }
  return MZGPU_OK;
}

int32_t mz_map_rows_dev(mzgpu_ctx* ctx, const u64* d_rows, u64 n, const mzgpu_closure* closure,
                        u64 skip_time, DevMem* out, u64* n_out) {
  *n_out = 0;
  MZ_TRY(out->alloc(ctx, n * 32));
  if (n == 0) return MZGPU_OK;
  const u64 n_tiles = (n + PT - 1) / PT;
  DevMem tiles;
  MZ_TRY(tiles.alloc(ctx, n_tiles * 4));
  u64* d_total = ctx->d_scratch + 29;
  mzgpu_closure cl;
  memset(&cl, 0, sizeof(cl));
  if (closure) cl = *closure;
  MZ_LAUNCH(ctx, (k_map_rows<false>), (unsigned)n_tiles, PT, 0, d_rows, n, cl, closure ? 1 : 0, skip_time,
            tiles.as<u32>(), (const u32*)nullptr, (u64*)nullptr);
  MZ_LAUNCH(ctx, k_scan_tiles, 1, 1024, 0, tiles.as<u32>(), n_tiles, d_total);
  MZ_LAUNCH(ctx, (k_map_rows<true>), (unsigned)n_tiles, PT, 0, d_rows, n, cl, closure ? 1 : 0, skip_time,
            (u32*)nullptr, tiles.as<u32>(), out->as<u64>());
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 29, d_total, 8, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 8;
  *n_out = ctx->h_scratch[29];
  return MZGPU_OK;
}

// ---------------------------------------------------------- single-pass forms
static unsigned lb_grid(mzgpu_ctx* ctx, u64 n_ub) {
  u64 tiles = (n_ub + PT - 1) / PT;
  u64 maxg = (u64)ctx->num_sms * 8;
  if (tiles > maxg) tiles = maxg;
  return (unsigned)(tiles ? tiles : 1);
}
// probes: tiles are handed out by ticket, so the grid only has to cover the machine
static unsigned probe_grid(mzgpu_ctx* ctx, u64 tiles) {
  u64 maxg = (u64)ctx->num_sms * 3;
  if (tiles > maxg) tiles = maxg;
  return (unsigned)(tiles ? tiles : 1);
}

int32_t mz_probe_async(mzgpu_ctx* ctx, const u64* d_stream, DLen n, u64 n_ub, const TraceView& trace,
                       const ProbeParams& pp, u64* d_out, DLen out_base, u64 out_cap, u64* d_out_len,
                       const MfpProbe* mfp) {
  LookBack lb;
  const u64 tiles = mz_probe_tiles(n_ub, trace.n_batches);
  const u32 tr = (u32)mz_probe_tile_rows(n_ub, trace.n_batches);
  MZ_TRY(mz_lookback_begin(ctx, tiles, &lb));
  const int out_rb = mfp != nullptr ? mfp->out_rb : pp.has_closure ? 32 : 40;
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * (32 + 16 * trace.n_batches + 32 + out_rb) : 0);  // exact counts only
  if (mfp != nullptr) {
    const MfpClosure cl = mfp_closure(*mfp, mfp->errs, mfp->err_cap, mfp->err_len);
    if (out_rb == 32) {
      MZ_LAUNCH(ctx, (k_probe_lb<4, MfpClosure>), probe_grid(ctx, tiles), PT, 0, d_stream, n, trace, pp, lb, d_out,
                out_base, out_cap, d_out_len, ctx->d_status, tr, cl);
    } else {
      MZ_LAUNCH(ctx, (k_probe_lb<5, MfpClosure>), probe_grid(ctx, tiles), PT, 0, d_stream, n, trace, pp, lb, d_out,
                out_base, out_cap, d_out_len, ctx->d_status, tr, cl);
    }
  } else if (pp.has_closure) {
    MZ_LAUNCH(ctx, (k_probe_lb<4>), probe_grid(ctx, tiles), PT, 0, d_stream, n, trace, pp, lb, d_out, out_base, out_cap,
              d_out_len, ctx->d_status, tr, BitClosure{});
  } else {
    MZ_LAUNCH(ctx, (k_probe_lb<5>), probe_grid(ctx, tiles), PT, 0, d_stream, n, trace, pp, lb, d_out, out_base, out_cap,
              d_out_len, ctx->d_status, tr, BitClosure{});
  }
  return MZGPU_OK;
}

// Several single-pass probes in one launch (see k_probe_chains).  jobs[j].chain: jobs of one chain
// are consecutive and share out / out_base / out_cap / out_len (taken from the chain's first job).
int32_t mz_probe_async_many(mzgpu_ctx* ctx, int k, const ProbeJobHost* jobs) {
  if (k <= 0) return MZGPU_OK;
  if (k > PROBE_MANY_MAX) {
    MZ_SET_ERR(ctx, "probe: %d jobs exceed the maximum %d per launch", k, PROBE_MANY_MAX);
    return MZGPU_E_INVALID;
  }
  static thread_local ProbeMany m;  // large: kept off the stack
  memset(&m, 0, sizeof(m));
  const bool closure = jobs[0].pp->has_closure != 0;
  const bool mfp = jobs[0].mfp != nullptr;
  const int out_rb = mfp ? jobs[0].mfp->out_rb : closure ? 32 : 40;
  ProbeClosures<MfpClosure> mcl;
  memset(&mcl, 0, sizeof(mcl));
  if (ctx->profile) {
    // per-kernel profiling: the algorithmic bytes of this launch need the actual stream lengths, which
    // live on the device -- one read-back ahead of the launch (outside its event bracket)
    bool pending = false;
    for (int j = 0; j < k; ++j) pending = pending || jobs[j].n.p != nullptr;
    if (pending) MZ_TRY(mz_resolve_counters(ctx));
  }
  u64 lb_at = 0, max_grid = 1, bytes = 0, total_tiles = 0, chain_tiles[PROBE_MANY_MAX] = {};
  int nc = 0;
  for (int j = 0; j < k; ++j) {
    if ((jobs[j].pp->has_closure != 0) != closure || (jobs[j].mfp != nullptr) != mfp ||
        (mfp && jobs[j].mfp->out_rb != out_rb)) {
      MZ_SET_ERR(ctx, "probe: jobs of one launch must agree on the output row shape");
      return MZGPU_E_INVALID;
    }
    m.job[j].stream = jobs[j].d_stream;
    m.job[j].dn = jobs[j].n;
    m.job[j].tv = *jobs[j].trace;
    m.job[j].pp = *jobs[j].pp;
    m.job[j].has_pre = jobs[j].has_pre ? 1 : 0;
    m.job[j].pre_has_closure = (jobs[j].has_pre && jobs[j].pre != nullptr) ? 1 : 0;
    m.job[j].skip_time = jobs[j].skip_time;
    if (m.job[j].pre_has_closure) m.job[j].pre = *jobs[j].pre;
    m.job[j].tile_rows = (u32)mz_probe_tile_rows(jobs[j].n_ub, jobs[j].trace->n_batches);
    if (mfp) mcl.c[j] = mfp_closure(*jobs[j].mfp, jobs[j].mfp->errs, jobs[j].mfp->err_cap, jobs[j].mfp->err_len);
    if (j == 0 || jobs[j].chain != jobs[j - 1].chain) {
      ProbeChain& c = m.chain[nc++];
      c.first = (u32)j;
      c.count = 0;
      c.out = jobs[j].d_out;
      c.out_base = jobs[j].out_base;
      c.out_cap = jobs[j].out_cap;
      c.out_len = jobs[j].d_out_len;
    }
    m.chain[nc - 1].count++;
  }
  m.n_chains = (u32)nc;
  for (int c = 0; c < nc; ++c) {
    u64 tiles = 0, rows_ub = 0;
    for (u32 q = 0; q < m.chain[c].count; ++q) {
      const ProbeJobHost& J = jobs[m.chain[c].first + q];
      tiles += mz_probe_tiles(J.n_ub, J.trace->n_batches);
      rows_ub += J.n_ub;
      u64 rows_now = J.n.imm;
      if (J.n.p != nullptr)  // (profiling only: the arena was just read back)
        rows_now = (ctx->profile && J.n.p >= ctx->d_cnt && J.n.p < ctx->d_cnt + (size_t)MZ_CNT_BLOCKS * 4) ? ctx->h_cnt[J.n.p - ctx->d_cnt] : 0;
      bytes += rows_now * (32 + 16 * J.trace->n_batches + 32 + out_rb);
    }
    MZ_TRY(mz_lookback_begin_at(ctx, lb_at, tiles, &m.chain[c].lb));
    lb_at += tiles;
    total_tiles += tiles;
    chain_tiles[c] = tiles;
  }
  // all chains of a launch run side by side: the resident CTAs (3 per SM) are shared out in proportion
  // to the chains' tiles
  const u64 resident = (u64)ctx->num_sms * 3;
  max_grid = 1;
  for (int c = 0; c < nc; ++c) {
    u64 g = total_tiles > 0 ? (resident * chain_tiles[c] + total_tiles - 1) / total_tiles : 1;
    if (g > chain_tiles[c]) g = chain_tiles[c];  // one CTA per tile at most
    if (g == 0) g = 1;                            // (an empty chain still has its length word to write)
    m.ctas[c] = (u32)g;
    if (g > max_grid) max_grid = g;
  }
  MZ_BYTES(ctx, bytes);
  if (mfp && out_rb == 32) {
    MZ_LAUNCH(ctx, (k_probe_chains<4, MfpClosure>), dim3((unsigned)max_grid, (unsigned)nc), PT, 0, m, ctx->d_status,
              mcl);
  } else if (mfp) {
    MZ_LAUNCH(ctx, (k_probe_chains<5, MfpClosure>), dim3((unsigned)max_grid, (unsigned)nc), PT, 0, m, ctx->d_status,
              mcl);
  } else if (closure) {
    MZ_LAUNCH(ctx, (k_probe_chains<4>), dim3((unsigned)max_grid, (unsigned)nc), PT, 0, m, ctx->d_status,
              ProbeClosures<BitClosure>{});
  } else {
    MZ_LAUNCH(ctx, (k_probe_chains<5>), dim3((unsigned)max_grid, (unsigned)nc), PT, 0, m, ctx->d_status,
              ProbeClosures<BitClosure>{});
  }
  return MZGPU_OK;
}

int32_t mz_map_rows_async(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const mzgpu_closure* closure,
                          u64 skip_time, u64* d_out, DLen out_base, u64 out_cap, u64* d_out_len) {
  LookBack lb;
  MZ_TRY(mz_lookback_begin(ctx, (n_ub + PT - 1) / PT, &lb));
  mzgpu_closure cl;
  memset(&cl, 0, sizeof(cl));
  if (closure) cl = *closure;
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * 64 : 0);
  MZ_LAUNCH(ctx, k_map_rows_lb, lb_grid(ctx, n_ub), PT, 0, d_rows, n, cl, closure ? 1 : 0, skip_time, lb, d_out,
            out_base, out_cap, d_out_len, ctx->d_status);
  return MZGPU_OK;
}
