// reduce.cu — accumulable reduce: COUNT / SUM moved into the diff (SURVEY.md a11-a12).
//
// Reference (src/compute/src/render/reduce.rs):
//   explode_one + datum_to_accumulator   :1313-1334, 1530-1669
//   Multiply<Diff> for Accum             :2043-2104
//   Semigroup for Accum (i128 wrapping)  :1940-2041
//   reduce_abelian closure + finalize    :1388-1409, 1671-1835
//   AccumulableErrorCheck                :1410-1466
//   FLOAT_SCALE = 2^24                   :1528
// and the reduce operator contract src/compute/src/extensions/reduce.rs:52-107.
//
// GPU shape: values become 80-byte accumulator rows (k_explode), the generic
// sort + segmented sum arranges them by (key, time), and k_corrections walks
// each changed key once: it sums the key's history from the prior batches of
// the arrangement (one hash probe per batch), then replays the new batch's
// times in order, emitting (-old, +new) output rows whenever the finalized
// aggregate changes.  All arithmetic is integer (i64 / i128 with carries), so
// results do not depend on summation order and match the reference bit for bit.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int RT = 256;

// (x * 2^24) as i128 with Rust's saturating float->int cast semantics.
__device__ __forceinline__ void f64_to_i128_sat(double x, u64* lo, u64* hi) {
  if (isnan(x)) {
    *lo = 0;
    *hi = 0;
    return;
  }
  const bool neg = x < 0.0;
  const double ax = fabs(x);
  if (ax < 9223372036854775808.0) {  // < 2^63: exact through i64 (truncation toward zero)
    long long v = (long long)x;
    *lo = (u64)v;
    *hi = v < 0 ? ~0ull : 0ull;
    return;
  }
  if (ax >= 170141183460469231731687303715884105728.0) {  // >= 2^127 (or inf): saturate
    if (neg) {
      *lo = 0;
      *hi = 0x8000000000000000ull;
    } else {
      *lo = ~0ull;
      *hi = 0x7fffffffffffffffull;
    }
    return;
  }
  const u64 bits = (u64)__double_as_longlong(ax);
  const int e = (int)((bits >> 52) & 0x7ff) - 1023;  // 63..126
  const u64 mant = (bits & 0xfffffffffffffull) | (1ull << 52);
  const int sh = e - 52;  // 11..74
  u64 l, h;
  if (sh >= 64) {
    l = 0;
    h = mant << (sh - 64);
  } else {
    l = mant << sh;
    h = mant >> (64 - sh);
  }
  if (neg) {  // two's complement negate
    l = ~l + 1;
    h = ~h + (l == 0 ? 1 : 0);
  }
  *lo = l;
  *hi = h;
}

// (i128 as f64): round to nearest, ties to even.
__device__ __forceinline__ double i128_to_f64(u64 lo, u64 hi) {
  const bool neg = (i64)hi < 0;
  if (neg) {
    lo = ~lo + 1;
    hi = ~hi + (lo == 0 ? 1 : 0);
  }
  double r;
  if (hi == 0) {
    r = __ull2double_rn(lo);
  } else {
    const int lz = __clzll((long long)hi);
    // top 64 bits of the 128-bit magnitude, sticky bit folded into bit 0
    const int shift = 64 - lz;  // bits shifted out of `lo`
    u64 top = lz == 0 ? hi : ((hi << lz) | (lo >> shift));
    u64 lost = lz == 0 ? lo : (lo << lz);
    if (lost) top |= 1;
    r = ldexp(__ull2double_rn(top), shift);
  }
  return neg ? -r : r;
}

// wrapping i128 * i64
__device__ __forceinline__ void mul_i128_i64(u64 lo, u64 hi, i64 d, u64* rlo, u64* rhi) {
  const u64 dl = (u64)d;
  const u64 dh = d < 0 ? ~0ull : 0ull;
  *rlo = lo * dl;
  *rhi = __umul64hi(lo, dl) + hi * dl + lo * dh;
}

// One lane of explode_one (datum_to_accumulator, reduce.rs:1530-1669): the lane's six diff words
// (non_nulls, acc_lo, acc_hi, pos_infs, neg_infs, nans) for value bits `v` and multiplicity `diff`.
// k_explode below computes the same words for its one column inline: written through this helper
// it compiles to a different register allocation, and the one-column kernel is kept as it was.
__device__ __forceinline__ void explode_lane(u64 v, bool f64, i64 diff, u64* o) {
  o[0] = (u64)diff;  // non_nulls
  u64 alo, ahi;
  u64 pinf = 0, ninf = 0, nan = 0;
  if (f64) {
    const double x = __longlong_as_double((long long)v);
    const bool is_nan = isnan(x);
    const bool is_pinf = isinf(x) && x > 0;
    const bool is_ninf = isinf(x) && x < 0;
    nan = is_nan ? (u64)diff : 0;
    pinf = is_pinf ? (u64)diff : 0;
    ninf = is_ninf ? (u64)diff : 0;
    if (is_nan || is_pinf || is_ninf) {
      alo = 0;
      ahi = 0;
    } else {
      f64_to_i128_sat(x * 16777216.0, &alo, &ahi);
    }
  } else {
    alo = v;
    ahi = (i64)v < 0 ? ~0ull : 0ull;
  }
  mul_i128_i64(alo, ahi, diff, &o[1], &o[2]);
  o[3] = pinf;
  o[4] = ninf;
  o[5] = nan;
}

__global__ void __launch_bounds__(RT) k_explode(const u64* __restrict__ rows, const DLen dn, int agg_kind,
                                                u64* __restrict__ out) {
  const u64 n = dlen_get(dn);
  for (u64 i = (u64)blockIdx.x * RT + threadIdx.x; i < n; i += (u64)gridDim.x * RT) {
  u64 r[4];
  load_row<4>(rows, i, r);
  const i64 diff = (i64)r[3];
  u64 o[10];
  o[0] = r[0];       // key
  o[1] = r[2];       // time
  o[2] = (u64)diff;  // total
  if (agg_kind == MZGPU_AGG_DISTINCT || agg_kind == MZGPU_AGG_THRESHOLD) {
    // only the multiplicity matters (build_distinct / threshold_arrangement)
#pragma unroll
    for (int w = 3; w < 10; ++w) o[w] = 0;
    store_row<10>(out, i, o);
    continue;
  }
  o[3] = (u64)diff;  // non_nulls
  u64 alo, ahi;
  u64 pinf = 0, ninf = 0, nan = 0;
  if (agg_kind == MZGPU_AGG_COUNT_SUM_F64) {
    const double v = __longlong_as_double((long long)r[1]);
    const bool is_nan = isnan(v);
    const bool is_pinf = isinf(v) && v > 0;
    const bool is_ninf = isinf(v) && v < 0;
    nan = is_nan ? (u64)diff : 0;
    pinf = is_pinf ? (u64)diff : 0;
    ninf = is_ninf ? (u64)diff : 0;
    if (is_nan || is_pinf || is_ninf) {
      alo = 0;
      ahi = 0;
    } else {
      f64_to_i128_sat(v * 16777216.0, &alo, &ahi);
    }
  } else {
    alo = r[1];
    ahi = (i64)r[1] < 0 ? ~0ull : 0ull;
  }
  mul_i128_i64(alo, ahi, diff, &o[4], &o[5]);
  o[6] = pinf;
  o[7] = ninf;
  o[8] = nan;
  o[9] = 0;
  store_row<10>(out, i, o);
  }
}

// a lane's value: the bit-field of its source word, sign-extended when asked
__device__ __forceinline__ u64 lane_value(const mzgpu_accum_lane& L, u64 key, u64 v1, u64 v2) {
  u64 v = field_get(L.field, key, v1, v2);
  if (L.sign_extend && L.field.bits < 64 && ((v >> (L.field.bits - 1)) & 1)) v |= ~0ull << L.field.bits;
  return v;
}

// explode_one of the lanes operator: R32 / R40 rows, lane l reads its bit-field of val1 / val2
template <int C>
__global__ void __launch_bounds__(RT) k_explode_lanes(const u64* __restrict__ rows, const DLen dn,
                                                      const __grid_constant__ LaneSet ls, u64* __restrict__ out) {
  constexpr int NW = LaneRows<C>::ARR_NW;
  const u64 n = dlen_get(dn);
  const u32 iw = ls.in_words;
  for (u64 i = (u64)blockIdx.x * RT + threadIdx.x; i < n; i += (u64)gridDim.x * RT) {
    const u64* r = rows + i * iw;
    const u64 key = r[0], v1 = r[1], v2 = iw == 5 ? r[2] : 0, t = r[iw - 2];
    const i64 diff = (i64)r[iw - 1];
    u64 o[NW];
    o[0] = key;
    o[1] = t;
    o[2] = (u64)diff;  // total
#pragma unroll
    for (int l = 0; l < C; ++l) {
      if ((u32)l < ls.n && ((ls.distinct_mask >> l) & 1u) == 0) {  // distinct lanes: mz_distinct_presence
        const mzgpu_accum_lane& L = ls.lane[l];
        explode_lane(lane_value(L, key, v1, v2), L.kind == MZGPU_AGG_COUNT_SUM_F64, diff, &o[3 + 6 * l]);
      } else {
#pragma unroll
        for (int w = 0; w < 6; ++w) o[3 + 6 * l + w] = 0;
      }
    }
#pragma unroll
    for (int w = 3 + 6 * C; w < NW; ++w) o[w] = 0;
    store_row<NW>(out, i, o);
  }
}

// finalize_accum + error-check flags for one accumulated diff S (the diff words of an arrangement
// row: total, then C lanes).  o = C x (count, sum_lo, sum_hi), flags.  For C = 1 the kind is
// agg_kind; for C >= 2 lane l is F64 if bit l of f64_mask is set, and lanes >= n_lanes (zero) get
// no flags.
template <int C>
__device__ __forceinline__ void finalize(const u64* S, int agg_kind, u32 f64_mask, u32 n_lanes, u64* o) {
  const i64 total = (i64)S[0];
  if (C == 1 && agg_kind == MZGPU_AGG_DISTINCT) {  // (key, ()) once; error flag for a negative multiplicity
    o[0] = 1;
    o[1] = 0;
    o[2] = 0;
    o[3] = total < 0 ? 2 : 0;
    return;
  }
  u64 flags = 0;
#pragma unroll
  for (int l = 0; l < C; ++l) {
    const u64* A = S + 1 + 6 * l;
    u64* q = o + 3 * l;
    const bool accum_zero = (A[0] | A[1] | A[2] | A[3] | A[4] | A[5]) == 0;
    u64 lf = 0;
    if (total > 0 && accum_zero) lf |= 1;
    if (total == 0 && !accum_zero) lf |= 2;
    if (C > 1 && (u32)l >= n_lanes) lf = 0;
    q[0] = A[0];
    const bool f64 = C == 1 ? agg_kind == MZGPU_AGG_COUNT_SUM_F64 : ((f64_mask >> l) & 1u) != 0;
    if (f64) {
      const i64 pinf = (i64)A[3], ninf = (i64)A[4], nan = (i64)A[5];
      u64 bits;
      if (nan > 0 || (pinf > 0 && ninf > 0))
        bits = 0x7ff8000000000000ull;
      else if (pinf > 0)
        bits = 0x7ff0000000000000ull;
      else if (ninf > 0)
        bits = 0xfff0000000000000ull;
      else
        bits = (u64)__double_as_longlong(i128_to_f64(A[1], A[2]) / 16777216.0);
      q[1] = bits;
      q[2] = 0;
    } else {
      q[1] = A[1];
      q[2] = A[2];
    }
    if (lf & 1) {
      q[1] = 0;
      q[2] = 0;
    }
    flags |= lf << (2 * l);
  }
  o[3 * C] = flags;
}

// ---------------------------------------------------------------- HAVING (mfp_after's filter)
// The predicate program of include/mzgpu.h (mzgpu_having), checked on the host (host.cu:
// validate_having), run on one finalized row.  Every thread of a warp reads the same ops from the
// parameter bank.  A stack value is (lo, hi): the i128 of an INT (sign-extended) or a NUM, the f64
// bits of a FLOAT (fl), 0 / 1 of a BOOL; st is HV_VAL, HV_NULL or HV_NULL + e for error e
// (MZGPU_HAVING_ERR_*, ordered as the EvalError variants, so the larger st is the larger error).
constexpr u32 HV_VAL = 0, HV_NULL = 1;

// OrderedFloat (Datum::Float64): NaN equals NaN and is above everything; -0.0 equals +0.0
__device__ __forceinline__ int hv_cmp3(u64 alo, u64 ahi, u64 blo, u64 bhi, bool fl) {
  if (fl) {
    const double a = __longlong_as_double((long long)alo), b = __longlong_as_double((long long)blo);
    const bool an = isnan(a), bn = isnan(b);
    if (an || bn) return an && bn ? 0 : (an ? 1 : -1);
    return a < b ? -1 : (a > b ? 1 : 0);
  }
  if (ahi != bhi) return (i64)ahi < (i64)bhi ? -1 : 1;
  return alo < blo ? -1 : (alo > blo ? 1 : 0);
}

// checked i64 arithmetic at SQL width w: add / sub / mul_int32 / 64 -> NumericFieldOverflow
// (src/expr/src/scalar/func.rs:107, 117, 690, 700, 904, 914); div_int32 / 64 truncates, DivisionByZero,
// MIN / -1 -> Int32OutOfRange / Int64OutOfRange (func.rs:1037-1059).  A 32-bit operation has int32
// operands (host-checked), so its exact result is the i64 one.  Returns 0 or the error.
__device__ __forceinline__ u32 hv_arith(int code, int w, i64 a, i64 b, i64* r) {
  i64 x;
  bool ovf = false;
  if (code == MZGPU_HOP_ADD) {
    x = (i64)((u64)a + (u64)b);
    ovf = ((a ^ x) & (b ^ x)) < 0;
  } else if (code == MZGPU_HOP_SUB) {
    x = (i64)((u64)a - (u64)b);
    ovf = ((a ^ b) & (a ^ x)) < 0;
  } else if (code == MZGPU_HOP_MUL) {
    x = (i64)((u64)a * (u64)b);
    ovf = __mul64hi((long long)a, (long long)b) != (x >> 63);
  } else {
    if (b == 0) return MZGPU_HAVING_ERR_DIVISION_BY_ZERO;
    if (b == -1 && a == (w == 32 ? (i64)(-2147483647 - 1) : (i64)0x8000000000000000ull))
      return w == 32 ? MZGPU_HAVING_ERR_INT32_OUT_OF_RANGE : MZGPU_HAVING_ERR_INT64_OUT_OF_RANGE;
    x = a / b;
  }
  if (w == 32 && x != (i64)(int)x) ovf = true;
  if (ovf) return MZGPU_HAVING_ERR_NUMERIC_FIELD_OVERFLOW;
  *r = x;
  return 0;
}

// The predicates on one finalized row v = C x (count, sum_lo, sum_hi), flags.  Returns the error
// (1..4) of the first predicate that raised one, 8 if every predicate is TRUE, 0 if one is FALSE or
// NULL (SafeMfpPlan::evaluate_inner, src/expr/src/linear.rs:1680-1700).
template <int C>
__device__ __forceinline__ u32 having_eval(const mzgpu_having& hv, u64 key, const u64* v, u32 f64_mask) {
  constexpr int D = MZGPU_HAVING_MAX_STACK;
  u64 lo[D], hi[D];
  u32 st[D];
  bool fl[D];
  for (u32 p = 0; p < hv.n_predicates; ++p) {
    int sp = 0;
    for (u32 i = 0; i < hv.n_ops[p]; ++i) {
      const mzgpu_having_op o = hv.ops[p][i];
      const u32 code = o.code;
      if (code <= MZGPU_HOP_FLOAT) {  // push
        u64 a = 0, b = 0;
        u32 s = HV_VAL;
        bool f = false;
        if (code == MZGPU_HOP_KEY) {
          a = key >> o.shift;
          if (o.bits < 64) {
            a &= (1ull << o.bits) - 1;
            if (o.sign_extend && ((a >> (o.bits - 1)) & 1)) a |= ~0ull << o.bits;
          }
          b = (i64)a < 0 ? ~0ull : 0;
        } else if (code == MZGPU_HOP_COUNT || code == MZGPU_HOP_SUM) {
#pragma unroll
          for (int l = 0; l < C; ++l) {  // (a select, not an index: v stays in registers)
            if ((u32)l != o.arg) continue;
            if (code == MZGPU_HOP_COUNT) {
              a = v[3 * l];
              b = (i64)a < 0 ? ~0ull : 0;
            } else {
              a = v[3 * l + 1];
              b = v[3 * l + 2];
              f = ((f64_mask >> l) & 1u) != 0;
              if ((v[3 * C] >> (2 * l)) & 1) s = HV_NULL;
            }
          }
        } else {
          a = hv.consts[o.konst].lo;
          b = hv.consts[o.konst].hi;
          f = code == MZGPU_HOP_FLOAT;
        }
        lo[sp] = a;
        hi[sp] = b;
        st[sp] = s;
        fl[sp] = f;
        ++sp;
        continue;
      }
      if (code == MZGPU_HOP_NOT) {
        if (st[sp - 1] == HV_VAL) lo[sp - 1] ^= 1;
        continue;
      }
      --sp;
      const int x = sp - 1, y = sp;  // x = the first operand and the result
      const u32 sx = st[x], sy = st[y];
      if (code == MZGPU_HOP_AND || code == MZGPU_HOP_OR) {
        // variadic And / Or (src/expr/src/scalar/func/variadic.rs:74-99, 1147-1170)
        const u64 dom = code == MZGPU_HOP_AND ? 0 : 1;
        if ((sx == HV_VAL && lo[x] == dom) || (sy == HV_VAL && lo[y] == dom)) {
          lo[x] = dom;
          st[x] = HV_VAL;
        } else {
          st[x] = sx > sy ? sx : sy;  // the larger error, else NULL, else both are the other value
        }
        continue;
      }
      if (sx > HV_NULL || sy > HV_NULL) {  // the first operand's error, else the second's
        st[x] = sx > HV_NULL ? sx : sy;
        continue;
      }
      if (sx == HV_NULL || sy == HV_NULL) {
        st[x] = HV_NULL;
        continue;
      }
      if (code == MZGPU_HOP_CMP) {
        const int c3 = hv_cmp3(lo[x], hi[x], lo[y], hi[y], fl[x]);
        bool r;
        switch (o.arg) {
          case MZGPU_CMP_EQ: r = c3 == 0; break;
          case MZGPU_CMP_NE: r = c3 != 0; break;
          case MZGPU_CMP_LT: r = c3 < 0; break;
          case MZGPU_CMP_LE: r = c3 <= 0; break;
          case MZGPU_CMP_GT: r = c3 > 0; break;
          default: r = c3 >= 0; break;
        }
        lo[x] = r ? 1 : 0;
        hi[x] = 0;
        fl[x] = false;
        continue;
      }
      i64 r = 0;
      const u32 e = hv_arith((int)code, o.arg, (i64)lo[x], (i64)lo[y], &r);
      if (e != 0) {
        st[x] = HV_NULL + e;
      } else {
        lo[x] = (u64)r;
        hi[x] = r < 0 ? ~0ull : 0;
      }
    }
    // one BOOL is left (host-checked)
    if (st[0] > HV_NULL) return st[0] - HV_NULL;
    if (st[0] == HV_NULL || lo[0] == 0) return 0;
  }
  return 8;
}

// Run the filter on a finalized row of a non-zero accumulation: its error goes into flag bits 16-18;
// returns whether the row is visible (a lane error flag, a predicate error, or every predicate TRUE).
template <int C>
__device__ __forceinline__ bool having_apply(const mzgpu_having& hv, u64 key, u64* v, u32 f64_mask) {
  const u32 r = having_eval<C>(hv, key, v, f64_mask);
  const u64 err = r & 7;
  v[3 * C] |= err << MZGPU_ROUT_HAVING_ERR_SHIFT;
  return err != 0 || (r & 8) != 0 || (v[3 * C] & 0xAAAAull) != 0;
}

// sum of all prior updates of `key` (times before the new batch).  The first hash
// slot of GROUP batches is fetched before any is inspected (independent loads).
template <int C>
__device__ __forceinline__ void prior_sum(const TraceView& tv, u64 key, u64* S) {
  constexpr int NW = LaneRows<C>::ARR_NW, ND = NW - 2;
  const u64 h0 = mix64(key);
  constexpr int GROUP = 8;
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
          const u64 bn = len != 0 ? first + len : bv_n(bv);
          for (u64 r = first; r < bn; ++r) {
            const u64* row = bv.rows + r * NW;
            if (len == 0 && row[0] != key) break;
            if (C == 1) {
              u64 d[ND];
#pragma unroll
              for (int w = 0; w < ND; ++w) d[w] = row[2 + w];
              diff_add<ND>(S, d);
            } else {
              diff_add<ND>(S, row + 2);  // wide rows: word by word from memory
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

// The corrections of ONE key, out[pos .. pos + c), put into consolidated order (the words after
// the key up to the time: C x (count, sum_lo, sum_hi), flags, time; the key is the same).  A key's
// corrections are distinct rows (-old and +new differ in their values, different times differ in
// the time word), and keys are written in ascending order by construction, so with this the
// kernel's whole output is already what consolidate() would return: the separate sort launch
// (40 us for a few hundred rows) is gone.
// Rows out[pos .. pos + c) of OW words sorted by their words 1 .. TWO (insertion sort: a key has a
// handful of corrections).
template <int OW, int TWO>
__device__ __forceinline__ void sort_run_rows(u64* __restrict__ out, u64 pos, u32 c) {
  for (u32 x = 1; x < c; ++x) {
    u64 r[OW];
    load_row<OW>(out, pos + x, r);
    u32 y = x;
    while (y > 0) {
      u64 p[OW];
      load_row<OW>(out, pos + y - 1, p);
      bool less = false;
#pragma unroll
      for (int w = 1; w <= TWO; ++w) {
        if (r[w] != p[w]) {
          less = r[w] < p[w];
          break;
        }
      }
      if (!less) break;
      store_row<OW>(out, pos + y, p);
      --y;
    }
    if (y != x) store_row<OW>(out, pos + y, r);
  }
}
template <int C>
__device__ __forceinline__ void sort_key_corrections(u64* __restrict__ out, u64 pos, u32 c) {
  sort_run_rows<LaneRows<C>::OUT_NW, LaneRows<C>::OUT_TW>(out, pos, c);
}

// output row (key, finalized aggregates, time, diff, zero padding)
template <int C>
__device__ __forceinline__ void put_out_row(u64* __restrict__ out, u64 at, u64 key, const u64* v, u64 t, u64 diff) {
  constexpr int OW = LaneRows<C>::OUT_NW, NV = 3 * C + 1;
  u64 r[OW];
  r[0] = key;
#pragma unroll
  for (int w = 0; w < NV; ++w) r[1 + w] = v[w];
  r[1 + NV] = t;
  r[2 + NV] = diff;
#pragma unroll
  for (int w = 3 + NV; w < OW; ++w) r[w] = 0;
  store_row<OW>(out, at, r);
}

// Corrections of one changed key: rows [i, ...) of the new batch with this key,
// given the key's prior accumulation S0.  Counts (and optionally writes at
// out[pos...]) the (-old, +new) output rows.  With HV the row exists only while the
// HAVING program `hv` lets it through (having_apply), and carries the program's error.
template <int C, bool HV = false>
__device__ __forceinline__ u32 walk_key(const u64* __restrict__ rows, u64 n, u64 i, u64 key, const u64* S0,
                                        int agg_kind, u32 f64_mask, u32 n_lanes, bool do_write,
                                        u64* __restrict__ out, u64 pos, const mzgpu_having* hv = nullptr) {
  constexpr int NW = LaneRows<C>::ARR_NW, ND = NW - 2, NV = 3 * C + 1;
  u64 S[ND];
#pragma unroll
  for (int w = 0; w < ND; ++w) S[w] = S0[w];
  if (C == 1 && agg_kind == MZGPU_AGG_THRESHOLD) {
    // output multiplicity = max(accumulated multiplicity, 0); one row per change, diff = the change
    i64 mult = (i64)S[0] > 0 ? (i64)S[0] : 0;
    u32 c = 0;
    for (u64 j = i; j < n; ++j) {
      const u64* row = rows + j * NW;
      if (row[0] != key) break;
      S[0] += row[2];
      const i64 m2 = (i64)S[0] > 0 ? (i64)S[0] : 0;
      if (m2 != mult) {
        if (do_write) {
          u64 r[8] = {key, 0, 0, 0, 0, row[1], (u64)(m2 - mult), 0};
          store_row<8>(out, pos + c, r);
        }
        ++c;
      }
      mult = m2;
    }
    if (do_write && c > 1) sort_key_corrections<C>(out, pos, c);
    return c;
  }
  bool had = !diff_is_zero<ND>(S);
  u64 oldv[NV];
#pragma unroll
  for (int w = 0; w < NV; ++w) oldv[w] = 0;
  if (had) finalize<C>(S, agg_kind, f64_mask, n_lanes, oldv);
  if constexpr (HV) {
    if (had) had = having_apply<C>(*hv, key, oldv, f64_mask);
  }
  u32 c = 0;
  for (u64 j = i; j < n; ++j) {
    const u64* row = rows + j * NW;
    if (row[0] != key) break;
    if (C == 1) {
      u64 d[ND];
#pragma unroll
      for (int w = 0; w < ND; ++w) d[w] = row[2 + w];
      diff_add<ND>(S, d);
    } else {
      diff_add<ND>(S, row + 2);
    }
    const u64 t = row[1];
    bool has = !diff_is_zero<ND>(S);
    u64 newv[NV];
#pragma unroll
    for (int w = 0; w < NV; ++w) newv[w] = 0;
    if (has) finalize<C>(S, agg_kind, f64_mask, n_lanes, newv);
    if constexpr (HV) {
      if (has) has = having_apply<C>(*hv, key, newv, f64_mask);
    }
    bool same = had && has;
#pragma unroll
    for (int w = 0; w < NV; ++w) same = same && oldv[w] == newv[w];
    if (!same) {
      if (had) {
        if (do_write) put_out_row<C>(out, pos + c, key, oldv, t, ~0ull);
        ++c;
      }
      if (has) {
        if (do_write) put_out_row<C>(out, pos + c, key, newv, t, 1);
        ++c;
      }
    }
    had = has;
#pragma unroll
    for (int w = 0; w < NV; ++w) oldv[w] = newv[w];
  }
  if (do_write && c > 1) sort_key_corrections<C>(out, pos, c);
  return c;
}

template <int C, bool WRITE>
__global__ void __launch_bounds__(RT) k_corrections(const u64* __restrict__ rows, u64 n,
                                                    const __grid_constant__ TraceView prior, int agg_kind,
                                                    u32 f64_mask, u32 n_lanes,
                                                    u32* __restrict__ tile_counts,
                                                    const u32* __restrict__ tile_base,
                                                    u64* __restrict__ out) {
  constexpr int NW = LaneRows<C>::ARR_NW, ND = NW - 2;
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * RT + threadIdx.x;
  u32 cnt = 0;
  const bool head = i < n && (i == 0 || rows[(i - 1) * NW] != rows[i * NW]);
  u64 key = 0;
  u64 S0[ND];
#pragma unroll
  for (int w = 0; w < ND; ++w) S0[w] = 0;
  if (head) {
    key = rows[i * NW];
    prior_sum<C>(prior, key, S0);
    cnt = walk_key<C>(rows, n, i, key, S0, agg_kind, f64_mask, n_lanes, false, nullptr, 0);
  }
  u32 total;
  u32 ex = block_exclusive_scan(cnt, sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
  } else {
    if (head && cnt > 0)
      walk_key<C>(rows, n, i, key, S0, agg_kind, f64_mask, n_lanes, true, out, (u64)tile_base[blockIdx.x] + ex);
  }
}

// single-pass form (sizes on the device, chained tiles): see probe.cu
template <int C>
__global__ void __launch_bounds__(RT) k_corrections_lb(const u64* __restrict__ rows, const DLen dn,
                                                       const __grid_constant__ TraceView prior, int agg_kind,
                                                       u32 f64_mask, u32 n_lanes,
                                                       const LookBack lb, u64* __restrict__ out, u64 out_cap,
                                                       u64* __restrict__ out_len, u64* __restrict__ status) {
  constexpr int NW = LaneRows<C>::ARR_NW, ND = NW - 2;
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  const u64 n = dlen_get(dn);
  const u64 n_tiles = (n + RT - 1) / RT;
  while (true) {
    const u32 tile = lb_next_tile(lb, &s_tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = 0;
      break;
    }
    const u64 i = (u64)tile * RT + threadIdx.x;
    u32 cnt = 0;
    const bool head = i < n && (i == 0 || rows[(i - 1) * NW] != rows[i * NW]);
    u64 key = 0;
    u64 S0[ND];
#pragma unroll
    for (int w = 0; w < ND; ++w) S0[w] = 0;
    if (head) {
      key = rows[i * NW];
      prior_sum<C>(prior, key, S0);
      cnt = walk_key<C>(rows, n, i, key, S0, agg_kind, f64_mask, n_lanes, false, nullptr, 0);
    }
    u32 total;
    const u32 ex = block_exclusive_scan(cnt, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &s_b);
    if (head && cnt > 0) {
      const u64 pos = excl + ex;
      if (pos + cnt > out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + cnt));
      else
        walk_key<C>(rows, n, i, key, S0, agg_kind, f64_mask, n_lanes, true, out, pos);
    }
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = excl + total;
  }
}

// The two forms above with a HAVING program (mzgpu_reduce_lanes_new_having).  They are separate kernels
// so that the unfiltered ones keep their code; the bounds are the same (at most two rows per new
// (key, time)), and sort_key_corrections keeps the output consolidated.
template <int C, bool WRITE>
__global__ void __launch_bounds__(RT) k_corrections_having(const u64* __restrict__ rows, u64 n,
                                                           const __grid_constant__ TraceView prior, u32 f64_mask,
                                                           u32 n_lanes, const __grid_constant__ mzgpu_having hv,
                                                           u32* __restrict__ tile_counts,
                                                           const u32* __restrict__ tile_base,
                                                           u64* __restrict__ out) {
  constexpr int NW = LaneRows<C>::ARR_NW, ND = NW - 2;
  // (the lanes operator: for C = 1 finalize takes lane 0's kind as the aggregate kind)
  const int agg_kind = (f64_mask & 1u) ? MZGPU_AGG_COUNT_SUM_F64 : MZGPU_AGG_COUNT_SUM_I64;
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * RT + threadIdx.x;
  u32 cnt = 0;
  const bool head = i < n && (i == 0 || rows[(i - 1) * NW] != rows[i * NW]);
  u64 key = 0;
  u64 S0[ND];
#pragma unroll
  for (int w = 0; w < ND; ++w) S0[w] = 0;
  if (head) {
    key = rows[i * NW];
    prior_sum<C>(prior, key, S0);
    cnt = walk_key<C, true>(rows, n, i, key, S0, agg_kind, f64_mask, n_lanes, false, nullptr, 0, &hv);
  }
  u32 total;
  u32 ex = block_exclusive_scan(cnt, sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
  } else {
    if (head && cnt > 0)
      walk_key<C, true>(rows, n, i, key, S0, agg_kind, f64_mask, n_lanes, true, out,
                        (u64)tile_base[blockIdx.x] + ex, &hv);
  }
}

template <int C>
__global__ void __launch_bounds__(RT) k_corrections_lb_having(const u64* __restrict__ rows, const DLen dn,
                                                              const __grid_constant__ TraceView prior, u32 f64_mask,
                                                              u32 n_lanes, const __grid_constant__ mzgpu_having hv,
                                                              const LookBack lb, u64* __restrict__ out, u64 out_cap,
                                                              u64* __restrict__ out_len, u64* __restrict__ status) {
  constexpr int NW = LaneRows<C>::ARR_NW, ND = NW - 2;
  const int agg_kind = (f64_mask & 1u) ? MZGPU_AGG_COUNT_SUM_F64 : MZGPU_AGG_COUNT_SUM_I64;
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  const u64 n = dlen_get(dn);
  const u64 n_tiles = (n + RT - 1) / RT;
  while (true) {
    const u32 tile = lb_next_tile(lb, &s_tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = 0;
      break;
    }
    const u64 i = (u64)tile * RT + threadIdx.x;
    u32 cnt = 0;
    const bool head = i < n && (i == 0 || rows[(i - 1) * NW] != rows[i * NW]);
    u64 key = 0;
    u64 S0[ND];
#pragma unroll
    for (int w = 0; w < ND; ++w) S0[w] = 0;
    if (head) {
      key = rows[i * NW];
      prior_sum<C>(prior, key, S0);
      cnt = walk_key<C, true>(rows, n, i, key, S0, agg_kind, f64_mask, n_lanes, false, nullptr, 0, &hv);
    }
    u32 total;
    const u32 ex = block_exclusive_scan(cnt, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &s_b);
    if (head && cnt > 0) {
      const u64 pos = excl + ex;
      if (pos + cnt > out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + cnt));
      else
        walk_key<C, true>(rows, n, i, key, S0, agg_kind, f64_mask, n_lanes, true, out, pos, &hv);
    }
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = excl + total;
  }
}
// the largest parameter block of the two (k_corrections_lb_having) within the classic 4 KB
static_assert(sizeof(TraceView) + sizeof(mzgpu_having) + sizeof(LookBack) + sizeof(DLen) + 6 * sizeof(u64) <= 4096,
              "k_corrections_lb_having parameters");

// ------------------------------------------------------------------ MIN / MAX
// Result of the hierarchical reduce (reduce.rs:1050-1135): per key the live
// (value, count) pairs; a negative count -> the error row, else MIN / MAX of the
// values.  One thread per changed key keeps the key's pairs in a small local table.
constexpr int MM_CAP = 32;
struct MinMaxAcc {
  u64 vals[MM_CAP];
  i64 cnts[MM_CAP];
  int m;
  bool overflow;
};
__device__ __forceinline__ void mm_add(MinMaxAcc& a, u64 val, i64 d) {
  for (int j = 0; j < a.m; ++j)
    if (a.vals[j] == val) {
      a.cnts[j] += d;
      return;
    }
  // reuse a dead entry before growing
  for (int j = 0; j < a.m; ++j)
    if (a.cnts[j] == 0) {
      a.vals[j] = val;
      a.cnts[j] = d;
      return;
    }
  if (a.m < MM_CAP) {
    a.vals[a.m] = val;
    a.cnts[a.m] = d;
    ++a.m;
  } else {
    a.overflow = true;
  }
}
__device__ __forceinline__ bool mm_eval(const MinMaxAcc& a, int agg_kind, u64* o /* count, sum_lo, sum_hi, flags */) {
  bool any = false, bad = false, have = false;
  u64 best = 0;
  for (int j = 0; j < a.m; ++j) {
    const i64 c = a.cnts[j];
    if (c == 0) continue;
    any = true;
    if (c < 0) {
      bad = true;
      continue;
    }
    const u64 v = a.vals[j];
    if (!have || (agg_kind == MZGPU_AGG_MIN ? v < best : v > best)) best = v;
    have = true;
  }
  o[0] = 0;
  o[1] = bad ? 0 : best;
  o[2] = 0;
  o[3] = bad ? 2 : 0;
  return any;
}
__device__ __forceinline__ void mm_prior(const TraceView& tv, u64 key, MinMaxAcc& a) {
  const u64 h0 = mix64(key);
  for (u32 b = 0; b < tv.n_batches; ++b) {
    const BatchView& bv = tv.b[b];
    const u64 mask = bv_mask(bv);
    u64 h = h0 & mask;
    while (true) {
      const ulonglong2 sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      if (sl.y == 0) break;
      if (sl.x == key) {
        const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
        const u32 len = (u32)(sl.y >> 44);
        const u64 bn = len != 0 ? first + len : bv_n(bv);
        for (u64 r = first; r < bn; ++r) {
          const ulonglong2* row = reinterpret_cast<const ulonglong2*>(bv.rows + r * 4);
          const ulonglong2 kv = row[0];
          if (len == 0 && kv.x != key) break;
          mm_add(a, kv.y, (i64)row[1].y);
        }
        break;
      }
      h = (h + 1) & mask;
    }
  }
}
// ---- groups wider than the local table (more than MM_CAP distinct live values of one key).
// The reference bounds the work per update with a tree of hashed buckets (build_bucketed,
// reduce.rs:796-900; top_k.rs:251-380); what the tree COMPUTES is the same per-key function of
// the key's (value, count) pairs.  Every batch holds a key's updates as a run sorted by (value,
// time), so that function is a k-way merge of the runs in value order, one value at a time --
// any group width, no table.  Only a key that overflowed the table takes this path.
struct RunCur {
  const u64* rows;
  u64 lo, hi;  // rows [lo, hi) of the key, sorted by (val, time)
};
constexpr int MM_MAX_RUNS = MZ_MAX_TRACE_BATCHES + 1;
// The key's run in every batch of `tv` (rows of NW words, sorted by key): one hash probe per batch.
template <int NW>
__device__ __forceinline__ int key_runs(const TraceView& tv, u64 key, RunCur* cur) {
  int nc = 0;
  const u64 h0 = mix64(key);
  for (u32 b = 0; b < tv.n_batches; ++b) {
    const BatchView& bv = tv.b[b];
    const u64 mask = bv_mask(bv);
    u64 h = h0 & mask;
    while (true) {
      const ulonglong2 sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      if (sl.y == 0) break;
      if (sl.x == key) {
        const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
        const u32 len = (u32)(sl.y >> 44);
        u64 end = first + len;
        if (len == 0) {  // run length not recorded: upper bound search (rows are sorted by key)
          u64 lo = first + 1, hi = bv_n(bv);
          while (lo < hi) {
            const u64 mid = (lo + hi) >> 1;
            if (bv.rows[mid * NW] == key)
              lo = mid + 1;
            else
              hi = mid;
          }
          end = lo;
        }
        cur[nc].rows = bv.rows;
        cur[nc].lo = first;
        cur[nc].hi = end;
        ++nc;
        break;
      }
      h = (h + 1) & mask;
    }
  }
  return nc;
}
__device__ __noinline__ int mm_runs(const TraceView& tv, u64 key, RunCur* cur) {
  int nc = 0;
  const u64 h0 = mix64(key);
  for (u32 b = 0; b < tv.n_batches; ++b) {
    const BatchView& bv = tv.b[b];
    const u64 mask = bv_mask(bv);
    u64 h = h0 & mask;
    while (true) {
      const ulonglong2 sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      if (sl.y == 0) break;
      if (sl.x == key) {
        const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
        const u32 len = (u32)(sl.y >> 44);
        u64 end = first + len;
        if (len == 0) {  // run length not recorded: upper bound search (rows are sorted by key)
          u64 lo = first + 1, hi = bv_n(bv);
          while (lo < hi) {
            const u64 mid = (lo + hi) >> 1;
            if (bv.rows[mid * 4] == key)
              lo = mid + 1;
            else
              hi = mid;
          }
          end = lo;
        }
        cur[nc].rows = bv.rows;
        cur[nc].lo = first;
        cur[nc].hi = end;
        ++nc;
        break;
      }
      h = (h + 1) & mask;
    }
  }
  return nc;
}
// Visit the key's distinct values in ascending (or descending) order with their total count:
// all rows of the prior runs, and the rows of the new batch's run [nlo, nhi) whose time is
// <= t_limit (use_new).  f(value, count) returns false to stop early.  The cursors are copied:
// `cur` is left untouched.
template <class F>
__device__ __forceinline__ void mm_stream(const RunCur* cur, int nc, const u64* nrows, u64 nlo, u64 nhi, bool use_new,
                                          u64 t_limit, bool desc, F f) {
  u64 lo[MM_MAX_RUNS], hi[MM_MAX_RUNS];
  for (int c = 0; c < nc; ++c) {
    lo[c] = cur[c].lo;
    hi[c] = cur[c].hi;
  }
  const int nn = use_new ? nc + 1 : nc;
  if (use_new) {
    lo[nc] = nlo;
    hi[nc] = nhi;
  }
  while (true) {
    bool have = false;
    u64 v = 0;
    for (int c = 0; c < nn; ++c) {
      if (lo[c] >= hi[c]) continue;
      const u64* rows = c < nc ? cur[c].rows : nrows;
      const u64 hv = rows[(desc ? hi[c] - 1 : lo[c]) * 4 + 1];
      if (!have || (desc ? hv > v : hv < v)) {
        v = hv;
        have = true;
      }
    }
    if (!have) break;
    i64 cnt = 0;
    for (int c = 0; c < nn; ++c) {
      const u64* rows = c < nc ? cur[c].rows : nrows;
      while (lo[c] < hi[c]) {
        const u64 r = desc ? hi[c] - 1 : lo[c];
        if (rows[r * 4 + 1] != v) break;
        if (c < nc || rows[r * 4 + 2] <= t_limit) cnt += (i64)rows[r * 4 + 3];
        if (desc)
          --hi[c];
        else
          ++lo[c];
      }
    }
    if (!f(v, cnt)) break;
  }
}
// The value words (1 .. NV) of a row of R32 (NV = 1) or R40 (NV = 2) input, compared as one unsigned tuple.
template <int NV>
__device__ __forceinline__ bool vals_less(const u64* a, const u64* b) {
  if (NV == 1) return a[0] < b[0];
  return a[0] != b[0] ? a[0] < b[0] : a[1] < b[1];
}
template <int NV>
__device__ __forceinline__ bool vals_eq(const u64* a, const u64* b) {
  return NV == 1 ? a[0] == b[0] : (a[0] == b[0] && a[1] == b[1]);
}
// mm_stream over rows of NW words (key, NW - 3 value words, time, diff), the distinct values compared as
// unsigned tuples: f(value, count) gets the word itself for R32 rows, a pointer to the value words otherwise.
// (mm_stream and mm_runs stay as they are: written through these templates, k_minmax_lb and walk_topk
// compile to different code.)
template <int NW, class F>
__device__ __forceinline__ void mm_stream_rows(const RunCur* cur, int nc, const u64* nrows, u64 nlo, u64 nhi, bool use_new,
                                          u64 t_limit, bool desc, F f) {
  constexpr int NV = NW - 3;
  u64 lo[MM_MAX_RUNS], hi[MM_MAX_RUNS];
  for (int c = 0; c < nc; ++c) {
    lo[c] = cur[c].lo;
    hi[c] = cur[c].hi;
  }
  const int nn = use_new ? nc + 1 : nc;
  if (use_new) {
    lo[nc] = nlo;
    hi[nc] = nhi;
  }
  while (true) {
    bool have = false;
    u64 v[NV];
#pragma unroll
    for (int w = 0; w < NV; ++w) v[w] = 0;
    for (int c = 0; c < nn; ++c) {
      if (lo[c] >= hi[c]) continue;
      const u64* rows = c < nc ? cur[c].rows : nrows;
      u64 hv[NV];
#pragma unroll
      for (int w = 0; w < NV; ++w) hv[w] = rows[(desc ? hi[c] - 1 : lo[c]) * NW + 1 + w];
      if (!have || (desc ? vals_less<NV>(v, hv) : vals_less<NV>(hv, v))) {
#pragma unroll
        for (int w = 0; w < NV; ++w) v[w] = hv[w];
        have = true;
      }
    }
    if (!have) break;
    i64 cnt = 0;
    for (int c = 0; c < nn; ++c) {
      const u64* rows = c < nc ? cur[c].rows : nrows;
      while (lo[c] < hi[c]) {
        const u64 r = desc ? hi[c] - 1 : lo[c];
        if (!vals_eq<NV>(rows + r * NW + 1, v)) break;
        if (c < nc || rows[r * NW + NW - 2] <= t_limit) cnt += (i64)rows[r * NW + NW - 1];
        if (desc)
          --hi[c];
        else
          ++lo[c];
      }
    }
    if constexpr (NV == 1) {
      if (!f(v[0], cnt)) break;
    } else {
      if (!f((const u64*)v, cnt)) break;
    }
  }
}
// MIN / MAX of a wide group: one ascending pass (every value is looked at: the error row needs
// to know about any negative count)
__device__ __noinline__ bool mm_eval_stream(const RunCur* cur, int nc, const u64* nrows, u64 nlo, u64 nhi, bool use_new,
                                            u64 t_limit, int agg_kind, u64* o) {
  bool any = false, bad = false, have = false;
  u64 best = 0;
  mm_stream(cur, nc, nrows, nlo, nhi, use_new, t_limit, false, [&](u64 v, i64 c) -> bool {
    if (c == 0) return true;
    any = true;
    if (c < 0) {
      bad = true;
      return true;
    }
    if (!have || agg_kind == MZGPU_AGG_MAX) best = v;  // ascending: first positive = MIN, last = MAX
    have = true;
    return true;
  });
  o[0] = 0;
  o[1] = bad ? 0 : best;
  o[2] = 0;
  o[3] = bad ? 2 : 0;
  return any;
}

// rows [i, ...) of the new batch share `key` (sorted by (val, time)): replay them in
// time order on top of the prior pairs and emit (-old, +new) whenever the result changes.
__device__ __noinline__ u32 walk_minmax(const u64* __restrict__ rows, u64 n, u64 i, u64 key,
                                        const TraceView& prior, int agg_kind, bool do_write,
                                        u64* __restrict__ out, u64 pos, u64* __restrict__ status) {
  MinMaxAcc a;
  a.m = 0;
  a.overflow = false;
  mm_prior(prior, key, a);
  // the key's run in the new batch, and (only if the table overflows) its runs in the prior batches
  u64 i_end = i;
  while (i_end < n && rows[i_end * 4] == key) ++i_end;
  RunCur runs[MM_MAX_RUNS];
  int n_runs = -1;
  auto eval_at = [&](bool use_new, u64 t_limit, u64* o) -> bool {
    if (!a.overflow) return mm_eval(a, agg_kind, o);
    if (n_runs < 0) n_runs = mm_runs(prior, key, runs);
    return mm_eval_stream(runs, n_runs, rows, i, i_end, use_new, t_limit, agg_kind, o);
  };
  u64 oldv[4];
  bool had = eval_at(false, 0, oldv);
  u32 c = 0;
  bool first = true;
  u64 t_prev = 0;
  while (true) {
    // next distinct time of this key
    bool found = false;
    u64 t_cur = 0;
    for (u64 j = i; j < n; ++j) {
      const u64* row = rows + j * 4;
      if (row[0] != key) break;
      const u64 t = row[2];
      if ((first || t > t_prev) && (!found || t < t_cur)) {
        t_cur = t;
        found = true;
      }
    }
    if (!found) break;
    for (u64 j = i; j < n; ++j) {
      const u64* row = rows + j * 4;
      if (row[0] != key) break;
      if (row[2] == t_cur) mm_add(a, row[1], (i64)row[3]);
    }
    u64 newv[4];
    const bool has = eval_at(true, t_cur, newv);
    const bool same = (had == has) && (!has || (oldv[1] == newv[1] && oldv[3] == newv[3]));
    if (!same) {
      if (had) {
        if (do_write) {
          u64 r[8] = {key, oldv[0], oldv[1], oldv[2], oldv[3], t_cur, ~0ull, 0};
          store_row<8>(out, pos + c, r);
        }
        ++c;
      }
      if (has) {
        if (do_write) {
          u64 r[8] = {key, newv[0], newv[1], newv[2], newv[3], t_cur, 1, 0};
          store_row<8>(out, pos + c, r);
        }
        ++c;
      }
    }
    had = has;
#pragma unroll
    for (int w = 0; w < 4; ++w) oldv[w] = newv[w];
    first = false;
    t_prev = t_cur;
  }
  (void)status;
  return c;
}

// ---------------------------------------------------------------------- TopK
// build_topk_negated_stage (top_k.rs:521-673): order the key's live values, skip `offset`
// rows, keep at most `limit` (multiplicities counted); a negative count -> the error row.
struct TopKWin {
  u64 v[MM_CAP];
  i64 m[MM_CAP];
  int n;
  bool err;
};
__device__ __noinline__ void tk_eval(const MinMaxAcc& a, const TopKParams& tp, TopKWin& w) {
  w.n = 0;
  w.err = false;
  for (int j = 0; j < a.m; ++j)
    if (a.cnts[j] < 0) {
      w.err = true;
      return;
    }
  u64 skip = tp.offset;
  i64 left = tp.limit;
  bool has_last = false;
  u64 last = 0;
  while (!(tp.limit >= 0 && left == 0)) {
    // next value in order (selection over at most MM_CAP live entries)
    int best = -1;
    for (int j = 0; j < a.m; ++j) {
      if (a.cnts[j] <= 0) continue;
      const u64 v = a.vals[j];
      const bool after = !has_last || (tp.descending ? v < last : v > last);
      if (after && (best < 0 || (tp.descending ? v > a.vals[best] : v < a.vals[best]))) best = j;
    }
    if (best < 0) break;
    last = a.vals[best];
    has_last = true;
    i64 cnt = a.cnts[best];
    if (skip > 0) {
      const u64 s = skip < (u64)cnt ? skip : (u64)cnt;
      skip -= s;
      cnt -= (i64)s;
    }
    if (tp.limit >= 0) {
      cnt = cnt < left ? cnt : left;
      left -= cnt;
    }
    if (cnt > 0) {
      w.v[w.n] = last;
      w.m[w.n] = cnt;
      ++w.n;
    }
  }
}
// the same window for a group wider than the table: a first pass looks for a negative count (the
// error row), a second walks the values in the plan's order until the limit is spent.  Returns
// false if the WINDOW itself has more than MM_CAP distinct values (limit > MM_CAP or none).
__device__ __noinline__ bool tk_eval_stream(const RunCur* cur, int nc, const u64* nrows, u64 nlo, u64 nhi, bool use_new,
                                            u64 t_limit, const TopKParams& tp, TopKWin& w) {
  w.n = 0;
  w.err = false;
  mm_stream(cur, nc, nrows, nlo, nhi, use_new, t_limit, false, [&](u64, i64 c) -> bool {
    if (c < 0) w.err = true;
    return !w.err;
  });
  if (w.err) return true;
  u64 skip = tp.offset;
  i64 left = tp.limit;
  bool fits = true;
  if (tp.limit == 0) return true;
  mm_stream(cur, nc, nrows, nlo, nhi, use_new, t_limit, tp.descending != 0, [&](u64 v, i64 c) -> bool {
    if (c <= 0) return true;
    i64 cnt = c;
    if (skip > 0) {
      const u64 s_ = skip < (u64)cnt ? skip : (u64)cnt;
      skip -= s_;
      cnt -= (i64)s_;
    }
    if (tp.limit >= 0) {
      cnt = cnt < left ? cnt : left;
      left -= cnt;
    }
    if (cnt > 0) {
      if (w.n == MM_CAP) {
        fits = false;
        return false;
      }
      w.v[w.n] = v;
      w.m[w.n] = cnt;
      ++w.n;
    }
    return !(tp.limit >= 0 && left == 0);
  });
  return fits;
}
// changes old -> fresh at time t; returns the number of rows (written at out[pos...] if do_write)
__device__ __forceinline__ u32 tk_emit(u64 key, const TopKWin& old, const TopKWin& fresh, u64 t, bool do_write,
                                       u64* __restrict__ out, u64 pos) {
  u32 c = 0;
  auto put = [&](u64 val, u64 flags, i64 d) {
    if (do_write) {
      u64 r[8] = {key, 0, val, 0, flags, t, (u64)d, 0};
      store_row<8>(out, pos + c, r);
    }
    ++c;
  };
  if (old.err != fresh.err) put(0, 2, fresh.err ? 1 : -1);
  for (int i = 0; i < old.n; ++i) {
    i64 now = 0;
    for (int j = 0; j < fresh.n; ++j)
      if (fresh.v[j] == old.v[i]) now = fresh.m[j];
    if (now != old.m[i]) put(old.v[i], 0, now - old.m[i]);
  }
  for (int j = 0; j < fresh.n; ++j) {
    bool seen = false;
    for (int i = 0; i < old.n; ++i) seen = seen || old.v[i] == fresh.v[j];
    if (!seen) put(fresh.v[j], 0, fresh.m[j]);
  }
  return c;
}
__device__ __noinline__ u32 walk_topk(const u64* __restrict__ rows, u64 n, u64 i, u64 key,
                                      const TraceView& prior, const TopKParams& tp, bool do_write,
                                      u64* __restrict__ out, u64 pos, u64* __restrict__ status) {
  MinMaxAcc a;
  a.m = 0;
  a.overflow = false;
  mm_prior(prior, key, a);
  u64 i_end = i;
  while (i_end < n && rows[i_end * 4] == key) ++i_end;
  RunCur runs[MM_MAX_RUNS];
  int n_runs = -1;
  bool window_fits = true;
  auto eval_at = [&](bool use_new, u64 t_limit, TopKWin& w) {
    if (!a.overflow) {
      tk_eval(a, tp, w);
      return;
    }
    if (n_runs < 0) n_runs = mm_runs(prior, key, runs);
    if (!tk_eval_stream(runs, n_runs, rows, i, i_end, use_new, t_limit, tp, w)) window_fits = false;
  };
  TopKWin old, fresh;
  eval_at(false, 0, old);
  u32 c = 0;
  bool first = true;
  u64 t_prev = 0;
  while (true) {
    bool found = false;
    u64 t_cur = 0;
    for (u64 j = i; j < n; ++j) {
      const u64* row = rows + j * 4;
      if (row[0] != key) break;
      const u64 t = row[2];
      if ((first || t > t_prev) && (!found || t < t_cur)) {
        t_cur = t;
        found = true;
      }
    }
    if (!found) break;
    for (u64 j = i; j < n; ++j) {
      const u64* row = rows + j * 4;
      if (row[0] != key) break;
      if (row[2] == t_cur) mm_add(a, row[1], (i64)row[3]);
    }
    eval_at(true, t_cur, fresh);
    c += tk_emit(key, old, fresh, t_cur, do_write, out, pos + c);
    old = fresh;
    first = false;
    t_prev = t_cur;
  }
  // (a window of more than MM_CAP distinct values -- LIMIT beyond 32 on a wide group -- is the one
  // shape still outside the subset: reported, never wrong)
  if (!window_fits) status[1] = 1;
  return c;
}

__global__ void __launch_bounds__(RT) k_minmax_lb(const u64* __restrict__ rows, const DLen dn,
                                                  const __grid_constant__ TraceView prior, int agg_kind,
                                                  const TopKParams tp, const LookBack lb,
                                                  u64* __restrict__ out, u64 out_cap,
                                                  u64* __restrict__ out_len, u64* __restrict__ status) {
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  const u64 n = dlen_get(dn);
  const u64 n_tiles = (n + RT - 1) / RT;
  const bool topk = agg_kind == MZGPU_AGG_TOPK;
  while (true) {
    const u32 tile = lb_next_tile(lb, &s_tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = 0;
      break;
    }
    const u64 i = (u64)tile * RT + threadIdx.x;
    u32 cnt = 0;
    const bool head = i < n && (i == 0 || rows[(i - 1) * 4] != rows[i * 4]);
    u64 key = 0;
    if (head) {
      key = rows[i * 4];
      cnt = topk ? walk_topk(rows, n, i, key, prior, tp, false, nullptr, 0, status)
                 : walk_minmax(rows, n, i, key, prior, agg_kind, false, nullptr, 0, status);
    }
    u32 total;
    const u32 ex = block_exclusive_scan(cnt, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &s_b);
    if (head && cnt > 0) {
      const u64 pos = excl + ex;
      if (pos + cnt > out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + cnt));
      else if (topk)
        walk_topk(rows, n, i, key, prior, tp, true, out, pos, status);
      else
        walk_minmax(rows, n, i, key, prior, agg_kind, true, out, pos, status);
    }
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = excl + total;
  }
}

// ------------------------------------------------------------ distinct lanes
// COUNT(DISTINCT x) / SUM(DISTINCT x) (build_accumulable's distinct_aggrs, reduce.rs:1338-1373): the input is
// mapped to ((key, value), ()) and arranged per lane ("Arranged Accumulable Distinct"); reduce_abelian emits
// ((key, value), +1) while the pair's accumulated multiplicity is non-zero, and explode_one turns each such
// output update into a diff vector with total = its diff and only this lane's Accum (that of the value).
// Here the pair arrangement is an R32 spine keyed by the group key, and k_distinct_presence emits those
// exploded rows for one new pair batch directly: one thread per (key, value) run of the batch.

struct PairMap {
  u64* out[MZGPU_MAX_ACCUM_LANES];  // R32 rows per distinct lane
  u64* len[MZGPU_MAX_ACCUM_LANES];  // where to write their row count, the input's (nullptr: known on the host)
  u32 lane[MZGPU_MAX_ACCUM_LANES];
  u32 k;
};
__global__ void __launch_bounds__(RT) k_distinct_pairs(const u64* __restrict__ rows, const DLen dn,
                                                       const __grid_constant__ LaneSet ls,
                                                       const __grid_constant__ PairMap pm) {
  const u64 n = dlen_get(dn);
  const u32 iw = ls.in_words;
  if (blockIdx.x == 0 && threadIdx.x < pm.k && pm.len[threadIdx.x] != nullptr) *pm.len[threadIdx.x] = n;
  for (u64 i = (u64)blockIdx.x * RT + threadIdx.x; i < n; i += (u64)gridDim.x * RT) {
    const u64* r = rows + i * iw;
    const u64 key = r[0], v1 = r[1], v2 = iw == 5 ? r[2] : 0;
    u64 o[4] = {key, 0, r[iw - 2], r[iw - 1]};
    for (u32 j = 0; j < pm.k; ++j) {
      o[1] = lane_value(ls.lane[pm.lane[j]], key, v1, v2);
      store_row<4>(pm.out[j], i, o);
    }
  }
}

// accumulated multiplicity of (key, val) over the prior batches of a pair arrangement: the key's rows come
// from the hash index (as mm_runs finds them), the value's rows inside them by binary search (R32 rows are
// sorted by (key, val, time))
__device__ __forceinline__ i64 pair_prior(const TraceView& tv, u64 key, u64 val) {
  i64 m = 0;
  const u64 h0 = mix64(key);
  for (u32 b = 0; b < tv.n_batches; ++b) {
    const BatchView& bv = tv.b[b];
    const u64 mask = bv_mask(bv);
    u64 h = h0 & mask;
    while (true) {
      const ulonglong2 sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      if (sl.y == 0) break;
      if (sl.x == key) {
        const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
        const u32 len = (u32)(sl.y >> 44);
        const u64 end = len != 0 ? first + len : bv_n(bv);  // (run length not recorded: the rows after it)
        u64 lo = first, hi = end;
        while (lo < hi) {  // first row with (key, val) >= (key, val)
          const u64 mid = (lo + hi) >> 1;
          const u64* x = bv.rows + mid * 4;
          if (x[0] < key || (x[0] == key && x[1] < val))
            lo = mid + 1;
          else
            hi = mid;
        }
        for (u64 r = lo; r < end; ++r) {
          const u64* x = bv.rows + r * 4;
          if (x[0] != key || x[1] != val) break;
          m += (i64)x[3];
        }
        break;
      }
      h = (h + 1) & mask;
    }
  }
  return m;
}

// The run of (key, val) at rows [i, ...) of the new pair batch, in time order on top of the prior
// multiplicity m: one class-C row (key, time, total = +-1, lane `lane` = the value's Accum times +-1) per
// change between zero and non-zero.  Returns the count; writes at out[pos ...] if do_write.
template <int C>
__device__ __forceinline__ u32 presence_walk(const u64* __restrict__ rows, u64 n, u64 i, u32 lane, i64 m,
                                             bool do_write, u64* __restrict__ out, u64 pos) {
  constexpr int NW = LaneRows<C>::ARR_NW;
  const u64 key = rows[i * 4], val = rows[i * 4 + 1];
  u32 c = 0;
  for (u64 j = i; j < n; ++j) {
    const u64* row = rows + j * 4;
    if (row[0] != key || row[1] != val) break;
    const bool was = m != 0;
    m += (i64)row[3];
    if (was == (m != 0)) continue;
    if (do_write) {
      const i64 s = was ? -1 : 1;
      u64 o[NW];
      o[0] = key;
      o[1] = row[2];
      o[2] = (u64)s;
#pragma unroll
      for (int l = 0; l < C; ++l) {
        if ((u32)l == lane) {
          explode_lane(val, false, s, &o[3 + 6 * l]);
        } else {
#pragma unroll
          for (int w = 0; w < 6; ++w) o[3 + 6 * l + w] = 0;
        }
      }
#pragma unroll
      for (int w = 3 + 6 * C; w < NW; ++w) o[w] = 0;
      store_row<NW>(out, pos + c, o);
    }
    ++c;
  }
  return c;
}

// The new pair batches of every distinct lane of an activation in one launch.  As in k_probe_chains, the
// tiles of the jobs are numbered one after the other (from the batch lengths on the device) and one
// look-back runs over all of them, so the rows of job q follow those of job q - 1.  A launch covers the
// tiles [tile0, tile0 + MZ_LB_TILES); the next launch continues at out_base = this launch's *out_len.
constexpr int DISTINCT_MAX = MZGPU_MAX_ACCUM_LANES;
struct DistinctJob {
  const u64* rows;
  DLen dn;
  u32 lane;
  TraceView prior;
};
struct DistinctMany {
  u32 k;
  DistinctJob job[DISTINCT_MAX];
};
static_assert(sizeof(DistinctMany) <= 32000, "kernel parameter space");

template <int C>
__global__ void __launch_bounds__(RT) k_distinct_presence(const __grid_constant__ DistinctMany m, u64 tile0,
                                                          const LookBack lb, const DLen out_base,
                                                          u64* __restrict__ out, u64 out_cap,
                                                          u64* __restrict__ out_len, u64* __restrict__ status) {
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  u64 nj[DISTINCT_MAX], tiles_before[DISTINCT_MAX + 1];
  tiles_before[0] = 0;
#pragma unroll
  for (int q = 0; q < DISTINCT_MAX; ++q) {
    nj[q] = (u32)q < m.k ? dlen_get(m.job[q].dn) : 0;
    tiles_before[q + 1] = tiles_before[q] + (nj[q] + RT - 1) / RT;
  }
  const u64 n_tiles = tiles_before[DISTINCT_MAX];
  const u64 tile_end = n_tiles < tile0 + MZ_LB_TILES ? n_tiles : tile0 + MZ_LB_TILES;
  const u64 base0 = dlen_get(out_base);
  while (true) {
    const u32 lt = lb_next_tile(lb, &s_tile);
    const u64 tile = tile0 + lt;
    if (tile >= tile_end) {
      if (lt == 0 && threadIdx.x == 0) *out_len = base0;  // no tile in this launch's range
      break;
    }
    u32 q = 0;
    while (q + 1 < m.k && tile >= tiles_before[q + 1]) ++q;
    const DistinctJob& J = m.job[q];
    const u64* rows = J.rows;
    const u64 n = nj[q];
    const u64 i = (tile - tiles_before[q]) * RT + threadIdx.x;
    const bool head =
        i < n && (i == 0 || rows[(i - 1) * 4] != rows[i * 4] || rows[(i - 1) * 4 + 1] != rows[i * 4 + 1]);
    u32 cnt = 0;
    i64 m0 = 0;
    if (head) {
      m0 = pair_prior(J.prior, rows[i * 4], rows[i * 4 + 1]);
      cnt = presence_walk<C>(rows, n, i, J.lane, m0, false, nullptr, 0);
    }
    u32 total;
    const u32 ex = block_exclusive_scan(cnt, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, lt, (u64)total, &s_b);
    if (head && cnt > 0) {
      const u64 pos = base0 + excl + ex;
      if (pos + cnt > out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + cnt));
      else
        presence_walk<C>(rows, n, i, J.lane, m0, true, out, pos);
    }
    if (tile == tile_end - 1 && threadIdx.x == 0) *out_len = base0 + excl + total;
  }
}

// ------------------------------------------------------------ monotonic MIN / MAX
// build_monotonic (reduce.rs:1138-1253) for append-only inputs: ensure_monotonic keeps a row iff its diff is
// positive (src/timely-util/src/operator.rs:425-456), the kept row's values move into the diff as one
// Min / Max monoid per aggregate, and the arrangement accumulates them (RowT<48> / RowT<112>, MZ_SG_MAX).
// Lane word = value ^ xm[l] (MonoXor): a max of the lane words is the lane's MIN or MAX, and the same xor
// decodes it.

// Input rows -> one arrangement row per row with diff > 0 (at arr[cnt[0]++]) and one R16 (time, +1) row per
// other row (at errs[cnt[1]++]); warp-aggregated slots, so the order within each output is arbitrary (the
// seal sorts the one, the error consolidation the other).
template <int C>
__global__ void __launch_bounds__(RT) k_monotonic_explode(const u64* __restrict__ rows, const DLen dn,
                                                          const __grid_constant__ LaneSet ls, const MonoXor mx,
                                                          u64* __restrict__ arr, u64* __restrict__ errs,
                                                          unsigned long long* __restrict__ cnt) {
  constexpr int NW = MonoRows<C>::ARR_NW;
  const u64 n = dlen_get(dn);
  const u32 iw = ls.in_words, lane = lane_id();
  for (u64 base = (u64)blockIdx.x * RT; base < n; base += (u64)gridDim.x * RT) {
    const u64 i = base + threadIdx.x;
    const bool valid = i < n;
    const u64* r = rows + (valid ? i : 0) * iw;
    const i64 diff = valid ? (i64)r[iw - 1] : 0;
    const bool ok = valid && diff > 0, bad = valid && diff <= 0;
    const u32 mok = __ballot_sync(0xffffffffu, ok), mbad = __ballot_sync(0xffffffffu, bad);
    unsigned long long bok = 0, bbad = 0;
    if (lane == 0) {
      if (mok) bok = atomicAdd(&cnt[0], (unsigned long long)__popc(mok));
      if (mbad) bbad = atomicAdd(&cnt[1], (unsigned long long)__popc(mbad));
    }
    bok = __shfl_sync(0xffffffffu, bok, 0);
    bbad = __shfl_sync(0xffffffffu, bbad, 0);
    const u32 lt = (1u << lane) - 1;
    if (ok) {
      const u64 key = r[0], v1 = r[1], v2 = iw == 5 ? r[2] : 0;
      u64 o[NW];
      o[0] = key;
      o[1] = r[iw - 2];
#pragma unroll
      for (int l = 0; l < C; ++l)
        o[2 + l] = (u32)l < ls.n ? lane_value(ls.lane[l], key, v1, v2) ^ mx.xm[l] : 0;
#pragma unroll
      for (int w = 2 + C; w < NW; ++w) o[w] = 0;
      store_row<NW>(arr, bok + __popc(mok & lt), o);
    }
    if (bad) {
      const u64 e[2] = {r[iw - 2], 1};
      store_row<2>(errs, bbad + __popc(mbad & lt), e);
    }
  }
}

// consolidate_named_if's data: the input rows with every value bit no lane reads cleared
__global__ void __launch_bounds__(RT) k_monotonic_mask(const u64* __restrict__ rows, const DLen dn, u32 iw, u64 m1,
                                                       u64 m2, u64* __restrict__ out) {
  const u64 n = dlen_get(dn);
  for (u64 i = (u64)blockIdx.x * RT + threadIdx.x; i < n; i += (u64)gridDim.x * RT) {
    const u64* r = rows + i * iw;
    u64* o = out + i * iw;
    for (u32 w = 0; w < iw; ++w) o[w] = r[w];
    o[1] &= m1;
    if (iw == 5) o[2] &= m2;
  }
}

// The key's accumulated lane words over the prior batches (max over its runs, one hash probe per batch);
// false if no batch holds the key.
template <int C>
__device__ __forceinline__ bool mono_prior(const TraceView& tv, u64 key, u64* S) {
  constexpr int NW = MonoRows<C>::ARR_NW, ND = NW - 2;
  const u64 h0 = mix64(key);
  bool found = false;
  for (u32 b = 0; b < tv.n_batches; ++b) {
    const BatchView& bv = tv.b[b];
    const u64 mask = bv_mask(bv);
    u64 h = h0 & mask;
    while (true) {
      const ulonglong2 sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      if (sl.y == 0) break;
      if (sl.x == key) {
        const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
        const u32 len = (u32)(sl.y >> 44);
        const u64 bn = len != 0 ? first + len : bv_n(bv);
        for (u64 r = first; r < bn; ++r) {
          const u64* row = bv.rows + r * NW;
          if (len == 0 && row[0] != key) break;
          diff_add<ND, MZ_SG_MAX>(S, row + 2);
          found = true;
        }
        break;
      }
      h = (h + 1) & mask;
    }
  }
  return found;
}

// output row (key, C decoded values, time, diff)
template <int C>
__device__ __forceinline__ void put_mono_row(u64* __restrict__ out, u64 at, u64 key, const u64* S, const MonoXor& mx,
                                             u64 t, u64 diff) {
  u64 r[MonoRows<C>::OUT_NW];
  r[0] = key;
#pragma unroll
  for (int l = 0; l < C; ++l) r[1 + l] = (u32)l < mx.n ? S[l] ^ mx.xm[l] : 0;
  r[1 + C] = t;
  r[2 + C] = diff;
  store_row<MonoRows<C>::OUT_NW>(out, at, r);
}

// The key's rows [i, ...) of the new batch in time order on top of its prior accumulation S0 (had: the key
// was in the arrangement): (-old, +new) whenever the accumulated lane words change, +new alone for the
// key's first row.  Returns the count; writes at out[pos ...], sorted, if do_write.
template <int C>
__device__ __forceinline__ u32 mono_walk(const u64* __restrict__ rows, u64 n, u64 i, u64 key, const u64* S0, bool had,
                                         const MonoXor& mx, bool do_write, u64* __restrict__ out, u64 pos) {
  constexpr int NW = MonoRows<C>::ARR_NW, ND = NW - 2;
  u64 S[ND];
#pragma unroll
  for (int w = 0; w < ND; ++w) S[w] = S0[w];
  u32 c = 0;
  for (u64 j = i; j < n; ++j) {
    const u64* row = rows + j * NW;
    if (row[0] != key) break;
    u64 T[ND];
#pragma unroll
    for (int w = 0; w < ND; ++w) T[w] = S[w];
    diff_add<ND, MZ_SG_MAX>(T, row + 2);
    bool same = had;
#pragma unroll
    for (int w = 0; w < ND; ++w) same = same && T[w] == S[w];
    if (!same) {
      if (had) {
        if (do_write) put_mono_row<C>(out, pos + c, key, S, mx, row[1], ~0ull);
        ++c;
      }
      if (do_write) put_mono_row<C>(out, pos + c, key, T, mx, row[1], 1);
      ++c;
    }
    had = true;
#pragma unroll
    for (int w = 0; w < ND; ++w) S[w] = T[w];
  }
  if (do_write && c > 1) sort_run_rows<MonoRows<C>::OUT_NW, C + 1>(out, pos, c);
  return c;
}

// the two-pass form (count, read back, write) for a batch past the single-pass bound
template <int C, bool WRITE>
__global__ void __launch_bounds__(RT) k_monotonic_corrections(const u64* __restrict__ rows, u64 n,
                                                              const __grid_constant__ TraceView prior, const MonoXor mx,
                                                              u32* __restrict__ tile_counts,
                                                              const u32* __restrict__ tile_base,
                                                              u64* __restrict__ out) {
  constexpr int NW = MonoRows<C>::ARR_NW, ND = NW - 2;
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * RT + threadIdx.x;
  u32 cnt = 0;
  const bool head = i < n && (i == 0 || rows[(i - 1) * NW] != rows[i * NW]);
  u64 key = 0;
  u64 S0[ND];
#pragma unroll
  for (int w = 0; w < ND; ++w) S0[w] = 0;
  bool had = false;
  if (head) {
    key = rows[i * NW];
    had = mono_prior<C>(prior, key, S0);
    cnt = mono_walk<C>(rows, n, i, key, S0, had, mx, false, nullptr, 0);
  }
  u32 total;
  const u32 ex = block_exclusive_scan(cnt, sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
  } else if (head && cnt > 0) {
    mono_walk<C>(rows, n, i, key, S0, had, mx, true, out, (u64)tile_base[blockIdx.x] + ex);
  }
}

// single-pass form (sizes on the device, chained tiles), as k_corrections_lb
template <int C>
__global__ void __launch_bounds__(RT) k_monotonic_corrections_lb(const u64* __restrict__ rows, const DLen dn,
                                                                 const __grid_constant__ TraceView prior,
                                                                 const MonoXor mx, const LookBack lb,
                                                                 u64* __restrict__ out, u64 out_cap,
                                                                 u64* __restrict__ out_len, u64* __restrict__ status) {
  constexpr int NW = MonoRows<C>::ARR_NW, ND = NW - 2;
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  const u64 n = dlen_get(dn);
  const u64 n_tiles = (n + RT - 1) / RT;
  while (true) {
    const u32 tile = lb_next_tile(lb, &s_tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = 0;
      break;
    }
    const u64 i = (u64)tile * RT + threadIdx.x;
    u32 cnt = 0;
    const bool head = i < n && (i == 0 || rows[(i - 1) * NW] != rows[i * NW]);
    u64 key = 0;
    u64 S0[ND];
#pragma unroll
    for (int w = 0; w < ND; ++w) S0[w] = 0;
    bool had = false;
    if (head) {
      key = rows[i * NW];
      had = mono_prior<C>(prior, key, S0);
      cnt = mono_walk<C>(rows, n, i, key, S0, had, mx, false, nullptr, 0);
    }
    u32 total;
    const u32 ex = block_exclusive_scan(cnt, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &s_b);
    if (head && cnt > 0) {
      const u64 pos = excl + ex;
      if (pos + cnt > out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + cnt));
      else
        mono_walk<C>(rows, n, i, key, S0, had, mx, true, out, pos);
    }
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = excl + total;
  }
}

// ------------------------------------------------------------ hierarchical MIN / MAX
// build_bucketed / build_bucketed_negated_output (reduce.rs:796-1135) over input that retracts: the
// arrangement holds the input rows masked to the bits the lanes read (key, val1[, val2], time | diff, an
// ordinary SUM diff).  Per key and time the output is every lane's MIN / MAX over the live rows while every
// live count is positive; a negative count puts the key in the error state instead (no row, one error).
// One thread per key run of the new batch keeps the key's distinct value rows in a local table; a key with
// more than MM_CAP of them takes the ordered merge of its runs (mm_stream), one pass per new time.
template <int NV>
struct HierAcc {
  u64 v[MM_CAP][NV];
  i64 c[MM_CAP];
  int m;
  bool overflow;
};
template <int NV>
__device__ __forceinline__ void hier_add(HierAcc<NV>& a, const u64* v, i64 d) {
  for (int j = 0; j < a.m; ++j)
    if (vals_eq<NV>(a.v[j], v)) {
      a.c[j] += d;
      return;
    }
  int at = -1;
  for (int j = 0; j < a.m && at < 0; ++j)  // reuse a dead entry before growing
    if (a.c[j] == 0) at = j;
  if (at < 0) {
    if (a.m == MM_CAP) {
      a.overflow = true;
      return;
    }
    at = a.m++;
  }
#pragma unroll
  for (int w = 0; w < NV; ++w) a.v[at][w] = v[w];
  a.c[at] = d;
}
// the key's rows in the prior batches (one hash probe per batch) into the table
template <int IW>
__device__ __forceinline__ void hier_prior(const TraceView& tv, u64 key, HierAcc<IW - 3>& a) {
  const u64 h0 = mix64(key);
  for (u32 b = 0; b < tv.n_batches && !a.overflow; ++b) {
    const BatchView& bv = tv.b[b];
    const u64 mask = bv_mask(bv);
    u64 h = h0 & mask;
    while (true) {
      const ulonglong2 sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      if (sl.y == 0) break;
      if (sl.x == key) {
        const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
        const u32 len = (u32)(sl.y >> 44);
        const u64 bn = len != 0 ? first + len : bv_n(bv);
        for (u64 r = first; r < bn; ++r) {
          const u64* row = bv.rows + r * IW;
          if (len == 0 && row[0] != key) break;
          hier_add<IW - 3>(a, row + 1, (i64)row[IW - 1]);
        }
        break;
      }
      h = (h + 1) & mask;
    }
  }
}
// one live value row folded into the lane words S (value ^ xm: a max of the words is the lane's MIN / MAX)
template <int C, int NV>
__device__ __forceinline__ void hier_fold(const LaneSet& ls, const MonoXor& mx, u64 key, const u64* v, u64* S) {
#pragma unroll
  for (int l = 0; l < C; ++l) {
    if ((u32)l >= ls.n) continue;
    const u64 w = lane_value(ls.lane[l], key, v[0], NV == 2 ? v[1] : 0) ^ mx.xm[l];
    S[l] = w > S[l] ? w : S[l];
  }
}
__device__ __forceinline__ const u64* hier_vals(const u64& v) { return &v; }
__device__ __forceinline__ const u64* hier_vals(const u64* v) { return v; }
constexpr u32 HIER_ROW = 1, HIER_ERR = 2;  // the key's state: it has an output row / it is in the error state

// The key's rows [i, ...) of the new batch (sorted by (values, time)) replayed in time order on top of its
// prior rows: (-old, +new) output rows whenever the lanes' values or the row's presence change, and an R32
// error row (key, 0, t, +1 entering / -1 leaving the error state) whenever that state changes.  Returns the
// output row count and the error row count (*n_err).  With do_write the output rows go to out[pos ...],
// sorted, and the error rows to errs[*err_len++] (a key's at most one error row per new time).
template <int IW, int C>
__device__ __noinline__ u32 hier_walk(const u64* __restrict__ rows, u64 n, u64 i, u64 key, const TraceView& prior,
                                      const LaneSet& ls, const MonoXor& mx, bool do_write, u64* __restrict__ out,
                                      u64 pos, u64* __restrict__ errs, u64 err_cap,
                                      unsigned long long* __restrict__ err_len, u64* __restrict__ status, u32* n_err) {
  constexpr int NV = IW - 3, TW = IW - 2, DW = IW - 1;
  HierAcc<NV> a;
  a.m = 0;
  a.overflow = false;
  hier_prior<IW>(prior, key, a);
  u64 i_end = i;
  while (i_end < n && rows[i_end * IW] == key) ++i_end;
  RunCur runs[MM_MAX_RUNS];
  int n_runs = -1;
  auto eval_at = [&](bool use_new, u64 t_limit, u64* S) -> u32 {
#pragma unroll
    for (int l = 0; l < C; ++l) S[l] = 0;
    bool any = false, bad = false;
    auto visit = [&](const u64* v, i64 c) {
      if (c == 0) return;
      any = true;
      if (c < 0)
        bad = true;
      else
        hier_fold<C, NV>(ls, mx, key, v, S);
    };
    if (!a.overflow) {
      for (int j = 0; j < a.m; ++j) visit(a.v[j], a.c[j]);
    } else {
      if (n_runs < 0) n_runs = key_runs<IW>(prior, key, runs);
      mm_stream_rows<IW>(runs, n_runs, rows, i, i_end, use_new, t_limit, false, [&](auto v, i64 c) -> bool {
        visit(hier_vals(v), c);
        return true;
      });
    }
    return bad ? HIER_ERR : (any ? HIER_ROW : 0);
  };
  u64 oldS[C];
  u32 olds = eval_at(false, 0, oldS);
  u32 c = 0, e = 0;
  bool first = true;
  u64 t_prev = 0;
  while (true) {
    // next distinct time of this key
    bool found = false;
    u64 t_cur = 0;
    for (u64 j = i; j < i_end; ++j) {
      const u64 t = rows[j * IW + TW];
      if ((first || t > t_prev) && (!found || t < t_cur)) {
        t_cur = t;
        found = true;
      }
    }
    if (!found) break;
    for (u64 j = i; j < i_end; ++j)
      if (rows[j * IW + TW] == t_cur) hier_add<NV>(a, rows + j * IW + 1, (i64)rows[j * IW + DW]);
    u64 newS[C];
    const u32 news = eval_at(true, t_cur, newS);
    const bool had = (olds & HIER_ROW) != 0, has = (news & HIER_ROW) != 0;
    bool same = had == has;
#pragma unroll
    for (int l = 0; l < C; ++l) same = same && (!has || oldS[l] == newS[l]);
    if (!same) {
      if (had) {
        if (do_write) put_mono_row<C>(out, pos + c, key, oldS, mx, t_cur, ~0ull);
        ++c;
      }
      if (has) {
        if (do_write) put_mono_row<C>(out, pos + c, key, newS, mx, t_cur, 1);
        ++c;
      }
    }
    if ((olds ^ news) & HIER_ERR) {
      if (do_write) {
        const u64 slot = atomicAdd(err_len, 1ull);
        const u64 r[4] = {key, 0, t_cur, (news & HIER_ERR) ? 1ull : ~0ull};
        if (slot < err_cap)
          store_row<4>(errs, slot, r);
        else
          atomicMax((unsigned long long*)status, (unsigned long long)(slot + 1));
      }
      ++e;
    }
    olds = news;
#pragma unroll
    for (int l = 0; l < C; ++l) oldS[l] = newS[l];
    first = false;
    t_prev = t_cur;
  }
  if (do_write && c > 1) sort_run_rows<MonoRows<C>::OUT_NW, C + 1>(out, pos, c);
  *n_err = e;
  return c;
}

// single-pass form (sizes on the device, chained tiles), as k_minmax_lb: one thread per key run of the new
// batch.  Output rows leave consolidated (keys ascending, each key's rows sorted by its thread); error rows
// leave in arbitrary order.
template <int IW, int C>
__global__ void __launch_bounds__(RT) k_hier_corrections_lb(const u64* __restrict__ rows, const DLen dn,
                                                            const __grid_constant__ TraceView prior,
                                                            const __grid_constant__ LaneSet ls, const MonoXor mx,
                                                            const LookBack lb, u64* __restrict__ out, u64 out_cap,
                                                            u64* __restrict__ out_len, u64* __restrict__ errs,
                                                            u64 err_cap, unsigned long long* __restrict__ err_len,
                                                            u64* __restrict__ status) {
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  const u64 n = dlen_get(dn);
  const u64 n_tiles = (n + RT - 1) / RT;
  while (true) {
    const u32 tile = lb_next_tile(lb, &s_tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = 0;
      break;
    }
    const u64 i = (u64)tile * RT + threadIdx.x;
    u32 cnt = 0, ecnt = 0;
    const bool head = i < n && (i == 0 || rows[(i - 1) * IW] != rows[i * IW]);
    u64 key = 0;
    if (head) {
      key = rows[i * IW];
      cnt = hier_walk<IW, C>(rows, n, i, key, prior, ls, mx, false, nullptr, 0, nullptr, 0, nullptr, nullptr, &ecnt);
    }
    u32 total;
    const u32 ex = block_exclusive_scan(cnt, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &s_b);
    if (head && (cnt > 0 || ecnt > 0)) {
      const u64 pos = excl + ex;
      if (pos + cnt > out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + cnt));
      else
        hier_walk<IW, C>(rows, n, i, key, prior, ls, mx, true, out, pos, errs, err_cap, err_len, status, &ecnt);
    }
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = excl + total;
  }
}

// the two-pass form (count, read back, write) for a batch past the single-pass bound; the error rows are
// written by the write pass
template <int IW, int C, bool WRITE>
__global__ void __launch_bounds__(RT) k_hier_corrections(const u64* __restrict__ rows, u64 n,
                                                         const __grid_constant__ TraceView prior,
                                                         const __grid_constant__ LaneSet ls, const MonoXor mx,
                                                         u32* __restrict__ tile_counts,
                                                         const u32* __restrict__ tile_base, u64* __restrict__ out,
                                                         u64* __restrict__ errs, u64 err_cap,
                                                         unsigned long long* __restrict__ err_len,
                                                         u64* __restrict__ status) {
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * RT + threadIdx.x;
  u32 cnt = 0, ecnt = 0;
  const bool head = i < n && (i == 0 || rows[(i - 1) * IW] != rows[i * IW]);
  u64 key = 0;
  if (head) {
    key = rows[i * IW];
    cnt = hier_walk<IW, C>(rows, n, i, key, prior, ls, mx, false, nullptr, 0, nullptr, 0, nullptr, nullptr, &ecnt);
  }
  u32 total;
  const u32 ex = block_exclusive_scan(cnt, sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
  } else if (head && (cnt > 0 || ecnt > 0)) {
    // (a pass with no output rows at all has no tile_base: it only writes error rows)
    const u64 pos = cnt > 0 ? (u64)tile_base[blockIdx.x] + ex : 0;
    hier_walk<IW, C>(rows, n, i, key, prior, ls, mx, true, out, pos, errs, err_cap, err_len, status, &ecnt);
  }
}

// ------------------------------------------------------------ monotonic TopK
// MonotonicTop1 / MonotonicTopK (src/compute/src/render/top_k.rs:102-214) for append-only inputs:
// ensure_monotonic keeps a row iff its diff is positive, and the arrangement holds only the window, the
// first `limit` units per key in order.  Window rows are RowT<72>: key, o0, o1, o2, val1, val2, time | diff.
constexpr int TK_NW = 9;

// the 72-byte row of input row r (to.in_words words) with diff `diff`, as k_topk_explode writes it (which keeps
// its own copy: calling this changed its generated code)
__device__ __forceinline__ void tk_encode(const TopKOrder& to, const u64* r, i64 diff, u64* o) {
  const u32 iw = to.in_words;
  const u64 key = r[0], v1 = r[1], v2 = iw == 5 ? r[2] : 0;
  o[0] = key;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    u64 v = 0;
    if ((u32)j < to.n) {
      v = field_get(to.f[j], key, v1, v2);
      const u32 bits = to.f[j].bits;
      if (to.sign_extend[j] && bits < 64 && ((v >> (bits - 1)) & 1)) v |= ~0ull << bits;
      v ^= to.xm[j];
    }
    o[1 + j] = v;
  }
  o[4] = v1;
  o[5] = v2;
  o[6] = r[iw - 2];
  o[7] = (u64)diff;
  o[8] = 0;
}

// Input rows -> one window row per row with diff > 0 (at arr[cnt[0]++]) and one R16 (time, +1) row per
// other row (at errs[cnt[1]++]); warp-aggregated slots, as k_monotonic_explode.
__global__ void __launch_bounds__(RT) k_topk_explode(const u64* __restrict__ rows, const DLen dn,
                                                     const __grid_constant__ TopKOrder to, u64* __restrict__ arr,
                                                     u64* __restrict__ errs, unsigned long long* __restrict__ cnt) {
  const u64 n = dlen_get(dn);
  const u32 iw = to.in_words, lane = lane_id();
  for (u64 base = (u64)blockIdx.x * RT; base < n; base += (u64)gridDim.x * RT) {
    const u64 i = base + threadIdx.x;
    const bool valid = i < n;
    const u64* r = rows + (valid ? i : 0) * iw;
    const i64 diff = valid ? (i64)r[iw - 1] : 0;
    const bool ok = valid && diff > 0, bad = valid && diff <= 0;
    const u32 mok = __ballot_sync(0xffffffffu, ok), mbad = __ballot_sync(0xffffffffu, bad);
    unsigned long long bok = 0, bbad = 0;
    if (lane == 0) {
      if (mok) bok = atomicAdd(&cnt[0], (unsigned long long)__popc(mok));
      if (mbad) bbad = atomicAdd(&cnt[1], (unsigned long long)__popc(mbad));
    }
    bok = __shfl_sync(0xffffffffu, bok, 0);
    bbad = __shfl_sync(0xffffffffu, bbad, 0);
    const u32 lt = (1u << lane) - 1;
    if (ok) {
      const u64 key = r[0], v1 = r[1], v2 = iw == 5 ? r[2] : 0;
      u64 o[TK_NW];
      o[0] = key;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        u64 v = 0;
        if ((u32)j < to.n) {
          v = field_get(to.f[j], key, v1, v2);
          const u32 bits = to.f[j].bits;
          if (to.sign_extend[j] && bits < 64 && ((v >> (bits - 1)) & 1)) v |= ~0ull << bits;
          v ^= to.xm[j];
        }
        o[1 + j] = v;
      }
      o[4] = v1;
      o[5] = v2;
      o[6] = r[iw - 2];
      o[7] = (u64)diff;
      o[8] = 0;
      store_row<TK_NW>(arr, bok + __popc(mok & lt), o);
    }
    if (bad) {
      const u64 e[2] = {r[iw - 2], 1};
      store_row<2>(errs, bbad + __popc(mbad & lt), e);
    }
  }
}

// the key's run in every batch of the window arrangement (one hash probe per batch); returns the count
__device__ __forceinline__ int tk_runs(const TraceView& tv, u64 key, u64* lo, u64* hi, uint8_t* bsel) {
  int nc = 0;
  const u64 h0 = mix64(key);
  for (u32 b = 0; b < tv.n_batches; ++b) {
    const BatchView& bv = tv.b[b];
    const u64 mask = bv_mask(bv);
    u64 h = h0 & mask;
    while (true) {
      const ulonglong2 sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      if (sl.y == 0) break;
      if (sl.x == key) {
        const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
        const u32 len = (u32)(sl.y >> 44);
        u64 end = first + len;
        if (len == 0) {  // run length not recorded: upper bound search (rows are sorted by key)
          u64 l = first + 1, r = bv_n(bv);
          while (l < r) {
            const u64 mid = (l + r) >> 1;
            if (bv.rows[mid * TK_NW] == key)
              l = mid + 1;
            else
              r = mid;
          }
          end = l;
        }
        lo[nc] = first;
        hi[nc] = end;
        bsel[nc] = (uint8_t)b;
        ++nc;
        break;
      }
      h = (h + 1) & mask;
    }
  }
  return nc;
}

// a < b on the row words 1..5 (o0, o1, o2, val1, val2): the order within a key
__device__ __forceinline__ bool tk_less(const u64* a, const u64* b) {
#pragma unroll
  for (int w = 1; w <= 5; ++w)
    if (a[w] != b[w]) return a[w] < b[w];
  return false;
}
__device__ __forceinline__ bool tk_same(const u64* a, const u64* b) {
  return a[1] == b[1] && a[2] == b[2] && a[3] == b[3] && a[4] == b[4] && a[5] == b[5];
}

// The window changes of one key whose new rows are nrows[i, nhi) (sorted by (row, time), consolidated,
// every diff positive).  The key's live window is the merge of its runs in the window arrangement, diffs
// summed.  The new rows are replayed one distinct time t at a time: the window at t is the first `limit`
// units of (window ∪ new rows with time <= t), so a row r holds min(units of r, limit - units before r),
// clamped at 0, and every row whose share changes from the previous time emits (r, t, change).  A pass
// stops where the units before reach the limit at the previous time: no row past that point is in either
// window, now or at any later time, so the next time is the least later time among the rows it visited.
// Returns the count; writes the window rows at win[pos ...] and the same rows at the input width (IW words)
// at out[pos ...], the latter sorted, if WRITE.
template <int IW, bool WRITE>
__device__ __noinline__ u32 tk_key(const TraceView& tv, const u64* __restrict__ nrows, u64 i, u64 nhi, u64 key,
                                   i64 limit, u64* __restrict__ win, u64* __restrict__ out, u64 pos) {
  if (limit == 0) return 0;
  u64 lo0[MM_MAX_RUNS], hi[MM_MAX_RUNS], lo[MM_MAX_RUNS];
  uint8_t bsel[MM_MAX_RUNS];
  // LIMIT NULL: every kept row enters, nothing is read
  const int nc = limit == INT64_MAX ? 0 : tk_runs(tv, key, lo0, hi, bsel);
  bool have_prev = false, have_cur = false;
  u64 tprev = 0, tcur = 0;
  u32 c = 0;
  while (true) {
    for (int k = 0; k < nc; ++k) lo[k] = lo0[k];
    u64 nlo = i;
    i64 cp = 0, cc = 0;  // units before the current row at the previous / current time
    bool have_next = false;
    u64 tnext = ~0ull;
    while (cp < limit) {
      const u64* best = nullptr;
      for (int k = 0; k < nc; ++k) {
        if (lo[k] >= hi[k]) continue;
        const u64* r = tv.b[bsel[k]].rows + lo[k] * TK_NW;
        if (best == nullptr || tk_less(r, best)) best = r;
      }
      if (nlo < nhi) {
        const u64* r = nrows + nlo * TK_NW;
        if (best == nullptr || tk_less(r, best)) best = r;
      }
      if (best == nullptr) break;
      u64 g[TK_NW];
      load_row<TK_NW>(best, 0, g);
      i64 o = 0, np = 0, ncur = 0;
      for (int k = 0; k < nc; ++k) {
        const u64* rows = tv.b[bsel[k]].rows;
        while (lo[k] < hi[k] && tk_same(rows + lo[k] * TK_NW, g)) {
          o += (i64)rows[lo[k] * TK_NW + 7];
          ++lo[k];
        }
      }
      while (nlo < nhi && tk_same(nrows + nlo * TK_NW, g)) {
        const u64 t = nrows[nlo * TK_NW + 6];
        const i64 d = (i64)nrows[nlo * TK_NW + 7];
        if (have_prev && t <= tprev) np += d;
        if (have_cur && t <= tcur) ncur += d;
        if ((!have_cur || t > tcur) && t < tnext) {
          tnext = t;
          have_next = true;
        }
        ++nlo;
      }
      const i64 mp = o + np, mc = o + ncur;
      const i64 wp = limit - cp <= 0 ? 0 : (mp < limit - cp ? mp : limit - cp);
      const i64 wc = limit - cc <= 0 ? 0 : (mc < limit - cc ? mc : limit - cc);
      if (have_cur && wc != wp) {
        if (WRITE) {
          g[0] = key;
          g[6] = tcur;
          g[7] = (u64)(wc - wp);
          g[8] = 0;
          store_row<TK_NW>(win, pos + c, g);
          u64 p[IW];
          p[0] = key;
          p[1] = g[4];
          if (IW == 5) p[2] = g[5];
          p[IW - 2] = tcur;
          p[IW - 1] = (u64)(wc - wp);
          store_row<IW>(out, pos + c, p);
        }
        ++c;
      }
      cp += mp;
      cc += mc;
    }
    if (!have_next) break;
    tprev = tcur;
    have_prev = have_cur;
    tcur = tnext;
    have_cur = true;
  }
  if (WRITE && c > 1) sort_run_rows<IW, IW - 2>(out, pos, c);
  return c;
}

// the key's new rows [i, end): end of its run in the new batch
__device__ __forceinline__ u64 tk_run_end(const u64* __restrict__ rows, u64 n, u64 i, u64 key) {
  u64 j = i + 1;
  while (j < n && rows[j * TK_NW] == key) ++j;
  return j;
}

// single-pass form (sizes on the device, chained tiles), as k_monotonic_corrections_lb: one thread per key
// run of the new rows
template <int IW>
__global__ void __launch_bounds__(RT) k_topk_window_lb(const u64* __restrict__ rows, const DLen dn,
                                                       const __grid_constant__ TraceView prior, const i64 limit,
                                                       const LookBack lb, u64* __restrict__ win, u64* __restrict__ out,
                                                       u64 out_cap, u64* __restrict__ out_len, u64* __restrict__ status) {
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  const u64 n = dlen_get(dn);
  const u64 n_tiles = (n + RT - 1) / RT;
  while (true) {
    const u32 tile = lb_next_tile(lb, &s_tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = 0;
      break;
    }
    const u64 i = (u64)tile * RT + threadIdx.x;
    u32 cnt = 0;
    const bool head = i < n && (i == 0 || rows[(i - 1) * TK_NW] != rows[i * TK_NW]);
    u64 key = 0, end = 0;
    if (head) {
      key = rows[i * TK_NW];
      end = tk_run_end(rows, n, i, key);
      cnt = tk_key<IW, false>(prior, rows, i, end, key, limit, nullptr, nullptr, 0);
    }
    u32 total;
    const u32 ex = block_exclusive_scan(cnt, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &s_b);
    if (head && cnt > 0) {
      const u64 pos = excl + ex;
      if (pos + cnt > out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + cnt));
      else
        tk_key<IW, true>(prior, rows, i, end, key, limit, win, out, pos);
    }
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = excl + total;
  }
}

// the two-pass form (count, read back, write) for a batch past the single-pass bound
template <int IW, bool WRITE>
__global__ void __launch_bounds__(RT) k_topk_window(const u64* __restrict__ rows, u64 n,
                                                    const __grid_constant__ TraceView prior, const i64 limit,
                                                    u32* __restrict__ tile_counts, const u32* __restrict__ tile_base,
                                                    u64* __restrict__ win, u64* __restrict__ out) {
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * RT + threadIdx.x;
  u32 cnt = 0;
  const bool head = i < n && (i == 0 || rows[(i - 1) * TK_NW] != rows[i * TK_NW]);
  u64 key = 0, end = 0;
  if (head) {
    key = rows[i * TK_NW];
    end = tk_run_end(rows, n, i, key);
    cnt = tk_key<IW, false>(prior, rows, i, end, key, limit, nullptr, nullptr, 0);
  }
  u32 total;
  const u32 ex = block_exclusive_scan(cnt, sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
  } else if (head && cnt > 0) {
    tk_key<IW, true>(prior, rows, i, end, key, limit, win, out, (u64)tile_base[blockIdx.x] + ex);
  }
}

// ------------------------------------------------------------ basic TopK
// BasicTopKPlan (build_topk_negated_stage, top_k.rs:521-673) over input that retracts: the input arrangement
// holds every input row as a 72-byte row with an ordinary SUM diff, and a negatives arrangement holds R32 rows
// (key, 0, time, delta) whose sum per key is the number of the key's rows with a negative accumulated count.

// Input rows -> one 72-byte row each, whatever its diff (row i at arr[i])
__global__ void __launch_bounds__(RT) k_topk_basic_explode(const u64* __restrict__ rows, const DLen dn,
                                                           const __grid_constant__ TopKOrder to, u64* __restrict__ arr) {
  const u64 n = dlen_get(dn);
  for (u64 i = (u64)blockIdx.x * RT + threadIdx.x; i < n; i += (u64)gridDim.x * RT) {
    const u64* r = rows + i * to.in_words;
    u64 o[TK_NW];
    tk_encode(to, r, (i64)r[to.in_words - 1], o);
    store_row<TK_NW>(arr, i, o);
  }
}

// the accumulated count of row g (words 1..5) in the key's prior runs [lo, hi): one lower-bound search per run
// (a run is sorted by (o0, o1, o2, val1, val2, time); before compaction a row may hold several times)
__device__ __forceinline__ i64 tkb_prior_count(const TraceView& tv, const u64* lo, const u64* hi,
                                               const uint8_t* bsel, int nc, const u64* g) {
  i64 s = 0;
  for (int k = 0; k < nc; ++k) {
    const u64* rows = tv.b[bsel[k]].rows;
    u64 l = lo[k], r = hi[k];
    while (l < r) {
      const u64 mid = (l + r) >> 1;
      if (tk_less(rows + mid * TK_NW, g))
        l = mid + 1;
      else
        r = mid;
    }
    for (; l < hi[k] && tk_same(rows + l * TK_NW, g); ++l) s += (i64)rows[l * TK_NW + 7];
  }
  return s;
}

// the key's negative-count rows before the new batch: the sum of its deltas in the negatives arrangement (R32
// rows; one hash probe per batch)
__device__ __forceinline__ i64 tkb_neg_prior(const TraceView& nv, u64 key) {
  i64 s = 0;
  const u64 h0 = mix64(key);
  for (u32 b = 0; b < nv.n_batches; ++b) {
    const BatchView& bv = nv.b[b];
    const u64 mask = bv_mask(bv);
    u64 h = h0 & mask;
    while (true) {
      const ulonglong2 sl = *reinterpret_cast<const ulonglong2*>(&bv.table[h]);
      if (sl.y == 0) break;
      if (sl.x == key) {
        const u64 first = (sl.y & MZ_SLOT_ROW_MASK) - 1;
        const u32 len = (u32)(sl.y >> 44);
        const u64 bn = len != 0 ? first + len : bv_n(bv);
        for (u64 r = first; r < bn && bv.rows[r * 4] == key; ++r) s += (i64)bv.rows[r * 4 + 3];
        break;
      }
      h = (h + 1) & mask;
    }
  }
  return s;
}

// the units of a row of m units with c units before it inside the window [off, end)
__device__ __forceinline__ i64 tkb_share(i64 c, i64 m, i64 off, i64 end) {
  const i64 a = c > off ? c : off;
  const i64 b = m > end - c ? end : c + m;
  return b > a ? b - a : 0;
}

// The changes of one key whose new rows are nrows[i, nhi) (sorted by (row, time), consolidated, any diff),
// replayed one distinct new time t at a time against its prior runs in the input arrangement:
//   (a) the key's negative-count rows at t: the negatives arrangement's count before the batch, plus, for each
//       touched row, whether its count (prior count by search, plus its new diffs <= t) is negative now and was
//       before.  A change emits (key, 0, t, delta) to `negs`; entering / leaving the error state (count > 0)
//       emits (key, 0, t, +1 / -1) to `errs`.  Both go to atomic slots (side_len[0] / [1], capacity side_cap;
//       an overflow is recorded in *status).
//   (b) the window changes from the previous time: an ordered merge of the prior runs with the new rows <= t,
//       a row's share the overlap of [before, before + count) with [offset, offset + limit), empty for a side
//       in the error state.  The walk stops once the units before the current row reach the window's end at
//       both times (counts can shrink, so one time's position bounds nothing).  Without a limit it stops at
//       the offset instead: past it every row is whole in both windows and only the new rows at t change,
//       unless the key enters or leaves the error state, which walks the whole window.
// Returns the output row count and the side row count (*n_side).  With WRITE the output rows (input width) go
// to out[pos ...], sorted.
template <int IW, bool WRITE>
__device__ __noinline__ u32 tkb_key(const TraceView& tv, const TraceView& nv, const u64* __restrict__ nrows, u64 i,
                                    u64 nhi, u64 key, i64 limit, i64 off, u64* __restrict__ out, u64 pos,
                                    u64* __restrict__ errs, u64* __restrict__ negs, u64 side_cap,
                                    unsigned long long* __restrict__ side_len, u64* __restrict__ status,
                                    u32* n_side) {
  u64 lo0[MM_MAX_RUNS], hi[MM_MAX_RUNS], lo[MM_MAX_RUNS];
  uint8_t bsel[MM_MAX_RUNS];
  const int nc = tk_runs(tv, key, lo0, hi, bsel);
  const bool no_limit = limit == INT64_MAX;
  const i64 end = no_limit ? INT64_MAX : off + limit;  // (the host refuses an overflowing offset + limit)
  const i64 n0 = tkb_neg_prior(nv, key);
  i64 nprev = n0;
  bool have_prev = false;
  u64 tprev = 0;
  u32 c = 0, e = 0;
  auto side = [&](u64* dst, int which, u64 t, i64 d) {
    if (WRITE) {
      const u64 slot = atomicAdd(&side_len[which], 1ull);
      const u64 r[4] = {key, 0, t, (u64)d};
      if (slot < side_cap)
        store_row<4>(dst, slot, r);
      else
        atomicMax((unsigned long long*)status, (unsigned long long)(slot + 1));
    }
    ++e;
  };
  auto emit = [&](const u64* g, u64 t, i64 d) {
    if (WRITE) {
      u64 p[IW];
      p[0] = key;
      p[1] = g[4];
      if (IW == 5) p[2] = g[5];
      p[IW - 2] = t;
      p[IW - 1] = (u64)d;
      store_row<IW>(out, pos + c, p);
    }
    ++c;
  };
  while (true) {
    bool found = false;
    u64 tcur = 0;
    for (u64 j = i; j < nhi; ++j) {
      const u64 t = nrows[j * TK_NW + 6];
      if ((!have_prev || t > tprev) && (!found || t < tcur)) {
        tcur = t;
        found = true;
      }
    }
    if (!found) break;
    // (a)
    i64 ncur = n0;
    for (u64 j = i; j < nhi;) {
      const u64* g = nrows + j * TK_NW;
      const i64 p = tkb_prior_count(tv, lo0, hi, bsel, nc, g);
      i64 s = p;
      for (; j < nhi && tk_same(nrows + j * TK_NW, g); ++j)
        if (nrows[j * TK_NW + 6] <= tcur) s += (i64)nrows[j * TK_NW + 7];
      ncur += (i64)(s < 0) - (i64)(p < 0);
    }
    const bool errp = nprev > 0, errc = ncur > 0;
    if (ncur != nprev) side(negs, 1, tcur, ncur - nprev);
    if (errp != errc) side(errs, 0, tcur, errc ? 1 : -1);
    // (b)
    if (limit > 0 && !(errp && errc)) {
      const bool tail = no_limit && !errp && !errc;
      const i64 stop = tail ? off : end;
      for (int k = 0; k < nc; ++k) lo[k] = lo0[k];
      u64 nlo = i;
      i64 cp = 0, cc = 0;  // units before the current row at the previous / current time
      while ((!errp && cp < stop) || (!errc && cc < stop)) {
        const u64* best = nullptr;
        for (int k = 0; k < nc; ++k) {
          if (lo[k] >= hi[k]) continue;
          const u64* r = tv.b[bsel[k]].rows + lo[k] * TK_NW;
          if (best == nullptr || tk_less(r, best)) best = r;
        }
        if (nlo < nhi) {
          const u64* r = nrows + nlo * TK_NW;
          if (best == nullptr || tk_less(r, best)) best = r;
        }
        if (best == nullptr) break;
        u64 g[TK_NW];
        load_row<TK_NW>(best, 0, g);
        i64 o = 0, np = 0, ncu = 0;
        for (int k = 0; k < nc; ++k) {
          const u64* rows = tv.b[bsel[k]].rows;
          while (lo[k] < hi[k] && tk_same(rows + lo[k] * TK_NW, g)) {
            o += (i64)rows[lo[k] * TK_NW + 7];
            ++lo[k];
          }
        }
        while (nlo < nhi && tk_same(nrows + nlo * TK_NW, g)) {
          const u64 t = nrows[nlo * TK_NW + 6];
          const i64 d = (i64)nrows[nlo * TK_NW + 7];
          if (have_prev && t <= tprev) np += d;
          if (t <= tcur) ncu += d;
          ++nlo;
        }
        const i64 mp = o + np, mc = o + ncu;
        const i64 wp = errp ? 0 : tkb_share(cp, mp, off, end), wc = errc ? 0 : tkb_share(cc, mc, off, end);
        if (wc != wp) emit(g, tcur, wc - wp);
        cp += mp;
        cc += mc;
      }
      if (tail)
        for (; nlo < nhi; ++nlo)
          if (nrows[nlo * TK_NW + 6] == tcur) emit(nrows + nlo * TK_NW, tcur, (i64)nrows[nlo * TK_NW + 7]);
    }
    nprev = ncur;
    tprev = tcur;
    have_prev = true;
  }
  if (WRITE && c > 1) sort_run_rows<IW, IW - 2>(out, pos, c);
  *n_side = e;
  return c;
}

// single-pass form (sizes on the device, chained tiles), as k_hier_corrections_lb: one thread per key run of
// the new rows.  Output rows leave consolidated; error and negatives rows leave in arbitrary order.
template <int IW>
__global__ void __launch_bounds__(RT) k_topk_basic_lb(const u64* __restrict__ rows, const DLen dn,
                                                      const __grid_constant__ TraceView prior,
                                                      const __grid_constant__ TraceView negv, const i64 limit,
                                                      const i64 off, const LookBack lb, u64* __restrict__ out,
                                                      u64 out_cap, u64* __restrict__ out_len, u64* __restrict__ errs,
                                                      u64* __restrict__ negs, u64 side_cap,
                                                      unsigned long long* __restrict__ side_len,
                                                      u64* __restrict__ status) {
  __shared__ u32 sm[34];
  __shared__ u32 s_tile;
  __shared__ u64 s_b;
  const u64 n = dlen_get(dn);
  const u64 n_tiles = (n + RT - 1) / RT;
  while (true) {
    const u32 tile = lb_next_tile(lb, &s_tile);
    if ((u64)tile >= n_tiles) {
      if (n_tiles == 0 && tile == 0 && threadIdx.x == 0) *out_len = 0;
      break;
    }
    const u64 i = (u64)tile * RT + threadIdx.x;
    u32 cnt = 0, ecnt = 0;
    const bool head = i < n && (i == 0 || rows[(i - 1) * TK_NW] != rows[i * TK_NW]);
    u64 key = 0, end = 0;
    if (head) {
      key = rows[i * TK_NW];
      end = tk_run_end(rows, n, i, key);
      cnt = tkb_key<IW, false>(prior, negv, rows, i, end, key, limit, off, nullptr, 0, nullptr, nullptr, 0, nullptr,
                               nullptr, &ecnt);
    }
    u32 total;
    const u32 ex = block_exclusive_scan(cnt, sm, &total);
    const u64 excl = lb_exclusive_prefix(lb, tile, (u64)total, &s_b);
    if (head && (cnt > 0 || ecnt > 0)) {
      const u64 pos = excl + ex;
      if (pos + cnt > out_cap)
        atomicMax((unsigned long long*)status, (unsigned long long)(pos + cnt));
      else
        tkb_key<IW, true>(prior, negv, rows, i, end, key, limit, off, out, pos, errs, negs, side_cap, side_len,
                          status, &ecnt);
    }
    if ((u64)tile == n_tiles - 1 && threadIdx.x == 0) *out_len = excl + total;
  }
}

// the two-pass form (count, read back, write) for a batch past the single-pass bound and for LIMIT NULL; the
// error and negatives rows are written by the write pass
template <int IW, bool WRITE>
__global__ void __launch_bounds__(RT) k_topk_basic(const u64* __restrict__ rows, u64 n,
                                                   const __grid_constant__ TraceView prior,
                                                   const __grid_constant__ TraceView negv, const i64 limit,
                                                   const i64 off, u32* __restrict__ tile_counts,
                                                   const u32* __restrict__ tile_base, u64* __restrict__ out,
                                                   u64* __restrict__ errs, u64* __restrict__ negs, u64 side_cap,
                                                   unsigned long long* __restrict__ side_len,
                                                   u64* __restrict__ status) {
  __shared__ u32 sm[34];
  const u64 i = (u64)blockIdx.x * RT + threadIdx.x;
  u32 cnt = 0, ecnt = 0;
  const bool head = i < n && (i == 0 || rows[(i - 1) * TK_NW] != rows[i * TK_NW]);
  u64 key = 0, end = 0;
  if (head) {
    key = rows[i * TK_NW];
    end = tk_run_end(rows, n, i, key);
    cnt = tkb_key<IW, false>(prior, negv, rows, i, end, key, limit, off, nullptr, 0, nullptr, nullptr, 0, nullptr,
                             nullptr, &ecnt);
  }
  u32 total;
  const u32 ex = block_exclusive_scan(cnt, sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
  } else if (head && (cnt > 0 || ecnt > 0)) {
    // (a pass with no output rows at all has no tile_base: it only writes error and negatives rows)
    const u64 pos = cnt > 0 ? (u64)tile_base[blockIdx.x] + ex : 0;
    tkb_key<IW, true>(prior, negv, rows, i, end, key, limit, off, out, pos, errs, negs, side_cap, side_len, status,
                      &ecnt);
  }
}

}  // namespace

// the grid of a launch over `tiles` tiles of RT rows: at most 8 blocks per SM (grid-stride or look-back loops)
static unsigned grid_of(mzgpu_ctx* ctx, u64 tiles) { return (unsigned)std::min<u64>(tiles, (u64)ctx->num_sms * 8); }

// Single-pass (look-back) correction kernels: the look-back state, the grid (at most 8 blocks per SM; at least
// one, which writes the length of no rows) and the bytes moved when the length is known on the host.
static int32_t lb_launch_setup(mzgpu_ctx* ctx, DLen n, u64 n_ub, u64 bytes_per_row, LookBack* lb, unsigned* grid) {
  const u64 tiles = (n_ub + RT - 1) / RT;
  MZ_TRY(mz_lookback_begin(ctx, tiles, lb));
  *grid = std::max(grid_of(ctx, tiles), 1u);
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * bytes_per_row : 0);
  return MZGPU_OK;
}

// Two-pass correction kernels over n > 0 rows: count(tile_counts, n_tiles) launches the count pass, one
// read-back of the scanned counts gives the total, alloc(total) makes the outputs, write(tile_base, n_tiles)
// launches the write pass if there are rows.
template <class Count, class Alloc, class Write>
static int32_t two_pass(mzgpu_ctx* ctx, u64 n, u64* n_out, Count count, Alloc alloc, Write write) {
  const u64 n_tiles = (n + RT - 1) / RT;
  DevMem tiles;
  MZ_TRY(tiles.alloc(ctx, n_tiles * 4));
  u64* d_total = ctx->d_scratch + 30;
  MZ_TRY(count(tiles.as<u32>(), n_tiles));
  MZ_LAUNCH(ctx, k_scan_tiles, 1, 1024, 0, tiles.as<u32>(), n_tiles, d_total);
  MZ_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 30, d_total, 8, cudaMemcpyDeviceToHost, ctx->stream));
  MZ_SYNC(ctx);
  ctx->stats.d2h_bytes += 8;
  const u64 total = ctx->h_scratch[30];
  MZ_TRY(alloc(total));
  *n_out = total;
  if (total == 0) return MZGPU_OK;
  return write((const u32*)tiles.as<u32>(), n_tiles);
}

int32_t mz_distinct_pairs(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const LaneSet& ls,
                          u64* const* d_pairs, u64* const* d_lens) {
  PairMap pm;
  memset(&pm, 0, sizeof(pm));
  for (u32 l = 0; l < ls.n; ++l) {
    if (((ls.distinct_mask >> l) & 1u) == 0) continue;
    pm.out[pm.k] = d_pairs[pm.k];
    pm.len[pm.k] = d_lens[pm.k];
    pm.lane[pm.k] = l;
    pm.k++;
  }
  const unsigned grid = std::max(grid_of(ctx, (n_ub + RT - 1) / RT), 1u);  // (the lengths are written for no rows)
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * (ls.in_words * 8 + 32 * pm.k) : 0);
  MZ_LAUNCH(ctx, k_distinct_pairs, grid, RT, 0, d_rows, n, ls, pm);
  return MZGPU_OK;
}

int32_t mz_distinct_presence(mzgpu_ctx* ctx, int c, int k, const DistinctJobHost* jobs, u64* d_out, u64 out_cap,
                             Lazy4* len, int* len_word) {
  if (k <= 0 || k > DISTINCT_MAX) {
    MZ_SET_ERR(ctx, "distinct presence: %d jobs (1..%d)", k, DISTINCT_MAX);
    return MZGPU_E_INVALID;
  }
  static thread_local DistinctMany m;  // large: kept off the stack
  memset(&m, 0, sizeof(m));
  m.k = (u32)k;
  u64 tiles = 0, bytes = 0;
  for (int j = 0; j < k; ++j) {
    m.job[j].rows = jobs[j].rows;
    m.job[j].dn = jobs[j].n;
    m.job[j].lane = jobs[j].lane;
    m.job[j].prior = *jobs[j].prior;
    tiles += (jobs[j].n_ub + RT - 1) / RT;
    if (jobs[j].n.p == nullptr) bytes += jobs[j].n.imm * (32 + 16 * jobs[j].prior->n_batches + mz_lane_arr_bytes(c));
  }
  MZ_TRY(len->make_pending(ctx));
  // one launch per MZ_LB_TILES tiles (the look-back state's size); each continues where the one before
  // stopped, with the running length alternating between two words of `len`
  const u64 launches = tiles > MZ_LB_TILES ? (tiles + MZ_LB_TILES - 1) / MZ_LB_TILES : 1;
  for (u64 x = 0; x < launches; ++x) {
    const u64 t0 = x * MZ_LB_TILES, lt = std::min<u64>(tiles - std::min(tiles, t0), MZ_LB_TILES);
    LookBack lb;
    MZ_TRY(mz_lookback_begin(ctx, lt, &lb));
    const unsigned grid = std::max(grid_of(ctx, lt), 1u);
    const DLen base = x == 0 ? dlen_imm(0) : DLen{len->dptr() + ((x - 1) & 1), 0};
    u64* out_len = len->dptr() + (x & 1);
    MZ_BYTES(ctx, x == 0 ? bytes : 0);
    MZ_TRY(mz_dispatch<LaneClasses>(ctx, c, "distinct presence", [&](auto C) {
      MZ_LAUNCH(ctx, k_distinct_presence<C>, grid, RT, 0, m, t0, lb, base, d_out, out_cap, out_len,
                ctx->d_status);
      return MZGPU_OK;
    }));
  }
  len->mark_written();
  *len_word = (int)((launches - 1) & 1);
  return MZGPU_OK;
}

// MIN / MAX / TopK corrections of a sealed R32 batch against the prior R32 arrangement.
// MIN / MAX: at most two output rows per distinct (key, time), capacity 2 * n_ub suffices;
// TopK: at most 2 * min(limit, 32) + 2 (every window entry may change, plus the error row).
int32_t mz_reduce_minmax_async(mzgpu_ctx* ctx, const u64* d_batch_rows, DLen n, u64 n_ub,
                               const TraceView& prior, int agg_kind, const TopKParams& tp, u64* d_out,
                               u64 out_cap, u64* d_out_len) {
  LookBack lb;
  unsigned grid;
  MZ_TRY(lb_launch_setup(ctx, n, n_ub, 32 + 16 + 32 + 128, &lb, &grid));
  MZ_LAUNCH(ctx, k_minmax_lb, grid, RT, 0, d_batch_rows, n, prior, agg_kind, tp, lb, d_out, out_cap,
            d_out_len, ctx->d_status);
  return MZGPU_OK;
}

int32_t mz_explode(mzgpu_ctx* ctx, const u64* d_r32, DLen n, u64 n_ub, int agg_kind, u64* d_racc) {
  if (n_ub == 0) return MZGPU_OK;
  const unsigned grid = grid_of(ctx, (n_ub + RT - 1) / RT);
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * 112 : 0);
  MZ_LAUNCH(ctx, k_explode, grid, RT, 0, d_r32, n, agg_kind, d_racc);
  return MZGPU_OK;
}

int32_t mz_explode_lanes(mzgpu_ctx* ctx, int c, const u64* d_rows, DLen n, u64 n_ub, const LaneSet& ls,
                         u64* d_arr) {
  if (n_ub == 0) return MZGPU_OK;
  const unsigned grid = grid_of(ctx, (n_ub + RT - 1) / RT);
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * (ls.in_words * 8 + mz_lane_arr_bytes(c)) : 0);
  return mz_dispatch<LaneClasses>(ctx, c, "explode", [&](auto C) {
    MZ_LAUNCH(ctx, k_explode_lanes<C>, grid, RT, 0, d_rows, n, ls, d_arr);
    return MZGPU_OK;
  });
}

int32_t mz_reduce_corrections(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, u64 n, const TraceView& prior,
                              int agg_kind, const LaneSet* ls, DevMem* out, u64* n_out, const mzgpu_having* hv) {
  *n_out = 0;
  if (n == 0) return out->alloc(ctx, 16);
  const u32 fm = ls != nullptr ? ls->f64_mask : 0, nl = ls != nullptr ? ls->n : 1;
  auto count = [&](u32* tile_counts, u64 n_tiles) {
    return mz_dispatch<LaneClasses>(ctx, c, "reduce", [&](auto C) {
      if (hv != nullptr)
        MZ_LAUNCH(ctx, (k_corrections_having<C, false>), (unsigned)n_tiles, RT, 0, d_batch_rows, n, prior, fm, nl,
                  *hv, tile_counts, (const u32*)nullptr, (u64*)nullptr);
      else
        MZ_LAUNCH(ctx, (k_corrections<C, false>), (unsigned)n_tiles, RT, 0, d_batch_rows, n, prior, agg_kind, fm, nl,
                  tile_counts, (const u32*)nullptr, (u64*)nullptr);
      return MZGPU_OK;
    });
  };
  auto alloc = [&](u64 total) { return out->alloc(ctx, total * mz_lane_out_bytes(c)); };
  auto write = [&](const u32* tile_base, u64 n_tiles) {
    return mz_dispatch<LaneClasses>(ctx, c, "reduce", [&](auto C) {
      if (hv != nullptr)
        MZ_LAUNCH(ctx, (k_corrections_having<C, true>), (unsigned)n_tiles, RT, 0, d_batch_rows, n, prior, fm, nl,
                  *hv, (u32*)nullptr, tile_base, out->as<u64>());
      else
        MZ_LAUNCH(ctx, (k_corrections<C, true>), (unsigned)n_tiles, RT, 0, d_batch_rows, n, prior, agg_kind, fm, nl,
                  (u32*)nullptr, tile_base, out->as<u64>());
      return MZGPU_OK;
    });
  };
  return two_pass(ctx, n, n_out, count, alloc, write);
}

// Single-pass form: batch length read on the device; at most two output rows per
// new (key, time) row, so capacity 2 * n_ub always suffices.
int32_t mz_reduce_corrections_async(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, DLen n, u64 n_ub,
                                    const TraceView& prior, int agg_kind, const LaneSet* ls, u64* d_out,
                                    u64 out_cap, u64* d_out_len, const mzgpu_having* hv) {
  const u32 fm = ls != nullptr ? ls->f64_mask : 0, nl = ls != nullptr ? ls->n : 1;
  LookBack lb;
  unsigned grid;
  MZ_TRY(lb_launch_setup(ctx, n, n_ub, 2 * mz_lane_arr_bytes(c) + 16 + 2 * mz_lane_out_bytes(c), &lb, &grid));
  return mz_dispatch<LaneClasses>(ctx, c, "reduce", [&](auto C) {
    if (hv != nullptr)
      MZ_LAUNCH(ctx, k_corrections_lb_having<C>, grid, RT, 0, d_batch_rows, n, prior, fm, nl, *hv, lb, d_out,
                out_cap, d_out_len, ctx->d_status);
    else
      MZ_LAUNCH(ctx, k_corrections_lb<C>, grid, RT, 0, d_batch_rows, n, prior, agg_kind, fm, nl, lb, d_out,
                out_cap, d_out_len, ctx->d_status);
    return MZGPU_OK;
  });
}

int32_t mz_monotonic_explode(mzgpu_ctx* ctx, int c, const u64* d_rows, DLen n, u64 n_ub, const LaneSet& ls,
                             const MonoXor& mx, u64* d_arr, u64* d_errs, u64* d_cnt) {
  MZ_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, 16, ctx->stream));
  if (n_ub == 0) return MZGPU_OK;
  const unsigned grid = grid_of(ctx, (n_ub + RT - 1) / RT);
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * (ls.in_words * 8 + mz_mono_arr_bytes(c)) : 0);
  return mz_dispatch<MonoClasses>(ctx, c, "monotonic explode", [&](auto C) {
    MZ_LAUNCH(ctx, k_monotonic_explode<C>, grid, RT, 0, d_rows, n, ls, mx, d_arr, d_errs,
              (unsigned long long*)d_cnt);
    return MZGPU_OK;
  });
}

int32_t mz_monotonic_mask(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, u32 in_words, u64 m1, u64 m2,
                          u64* d_out) {
  if (n_ub == 0) return MZGPU_OK;
  const unsigned grid = grid_of(ctx, (n_ub + RT - 1) / RT);
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * in_words * 16 : 0);
  MZ_LAUNCH(ctx, k_monotonic_mask, grid, RT, 0, d_rows, n, in_words, m1, m2, d_out);
  return MZGPU_OK;
}

// at most two output rows per new (key, time) row: capacity 2 * n_ub suffices
int32_t mz_monotonic_corrections_async(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, DLen n, u64 n_ub,
                                       const TraceView& prior, const MonoXor& mx, u64* d_out, u64 out_cap,
                                       u64* d_out_len) {
  LookBack lb;
  unsigned grid;
  MZ_TRY(lb_launch_setup(ctx, n, n_ub, 2 * mz_mono_arr_bytes(c) + 16 + 2 * mz_mono_out_bytes(c), &lb, &grid));
  return mz_dispatch<MonoClasses>(ctx, c, "monotonic reduce", [&](auto C) {
    MZ_LAUNCH(ctx, k_monotonic_corrections_lb<C>, grid, RT, 0, d_batch_rows, n, prior, mx, lb, d_out,
              out_cap, d_out_len, ctx->d_status);
    return MZGPU_OK;
  });
}

int32_t mz_monotonic_corrections(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, u64 n, const TraceView& prior,
                                 const MonoXor& mx, DevMem* out, u64* n_out) {
  *n_out = 0;
  if (n == 0) return out->alloc(ctx, 16);
  auto count = [&](u32* tile_counts, u64 n_tiles) {
    return mz_dispatch<MonoClasses>(ctx, c, "monotonic reduce", [&](auto C) {
      MZ_LAUNCH(ctx, (k_monotonic_corrections<C, false>), (unsigned)n_tiles, RT, 0, d_batch_rows, n, prior, mx,
                tile_counts, (const u32*)nullptr, (u64*)nullptr);
      return MZGPU_OK;
    });
  };
  auto alloc = [&](u64 total) { return out->alloc(ctx, total * mz_mono_out_bytes(c)); };
  auto write = [&](const u32* tile_base, u64 n_tiles) {
    return mz_dispatch<MonoClasses>(ctx, c, "monotonic reduce", [&](auto C) {
      MZ_LAUNCH(ctx, (k_monotonic_corrections<C, true>), (unsigned)n_tiles, RT, 0, d_batch_rows, n, prior, mx,
                (u32*)nullptr, tile_base, out->as<u64>());
      return MZGPU_OK;
    });
  };
  return two_pass(ctx, n, n_out, count, alloc, write);
}

struct InRowWords : IntSet<4, 5> {  // R32 / R40 input
  static constexpr const char* kind = "input row words";
};

// the hierarchical reduce's kernels for the input width (ls.in_words) and lane class c
template <class F>
static int32_t hier_dispatch(mzgpu_ctx* ctx, int c, const LaneSet& ls, F&& f) {
  return mz_dispatch<InRowWords>(ctx, (int)ls.in_words, "hierarchical reduce", [&](auto IW) {
    return mz_dispatch<MonoClasses>(ctx, c, "hierarchical reduce", [&](auto C) { return f(IW, C); });
  });
}

// at most two output rows and one error row per new (key, time) row: capacities 2 * n_ub and n_ub suffice
int32_t mz_hier_corrections_async(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, DLen n, u64 n_ub,
                                  const TraceView& prior, const LaneSet& ls, const MonoXor& mx, u64* d_out,
                                  u64 out_cap, u64* d_out_len, u64* d_errs, u64 err_cap, u64* d_err_len) {
  MZ_CUDA(ctx, cudaMemsetAsync(d_err_len, 0, 8, ctx->stream));
  LookBack lb;
  unsigned grid;
  MZ_TRY(lb_launch_setup(ctx, n, n_ub, 2 * ls.in_words * 8 + 2 * mz_mono_out_bytes(c), &lb, &grid));
  return hier_dispatch(ctx, c, ls, [&](auto IW, auto C) {
    MZ_LAUNCH(ctx, (k_hier_corrections_lb<IW, C>), grid, RT, 0, d_batch_rows, n, prior, ls, mx, lb, d_out, out_cap,
              d_out_len, d_errs, err_cap, (unsigned long long*)d_err_len, ctx->d_status);
    return MZGPU_OK;
  });
}

int32_t mz_hier_corrections(mzgpu_ctx* ctx, int c, const u64* d_batch_rows, u64 n, const TraceView& prior,
                            const LaneSet& ls, const MonoXor& mx, DevMem* out, u64* n_out, u64* d_errs, u64 err_cap,
                            u64* d_err_len) {
  *n_out = 0;
  MZ_CUDA(ctx, cudaMemsetAsync(d_err_len, 0, 8, ctx->stream));
  if (n == 0) return out->alloc(ctx, 16);
  auto count = [&](u32* tile_counts, u64 n_tiles) {
    return hier_dispatch(ctx, c, ls, [&](auto IW, auto C) {
      MZ_LAUNCH(ctx, (k_hier_corrections<IW, C, false>), (unsigned)n_tiles, RT, 0, d_batch_rows, n, prior, ls, mx,
                tile_counts, (const u32*)nullptr, (u64*)nullptr, (u64*)nullptr, (u64)0, (unsigned long long*)nullptr,
                ctx->d_status);
      return MZGPU_OK;
    });
  };
  auto alloc = [&](u64 total) { return out->alloc(ctx, std::max<u64>(total, 1) * mz_mono_out_bytes(c)); };
  auto write = [&](const u32* tile_base, u64 n_tiles) {
    return hier_dispatch(ctx, c, ls, [&](auto IW, auto C) {
      MZ_LAUNCH(ctx, (k_hier_corrections<IW, C, true>), (unsigned)n_tiles, RT, 0, d_batch_rows, n, prior, ls, mx,
                (u32*)nullptr, tile_base, out->as<u64>(), d_errs, err_cap, (unsigned long long*)d_err_len,
                ctx->d_status);
      return MZGPU_OK;
    });
  };
  const u64 n_tiles = (n + RT - 1) / RT;
  MZ_TRY(two_pass(ctx, n, n_out, count, alloc, write));
  // a batch whose keys change no output row can still move keys into or out of the error state
  if (*n_out == 0) return write(nullptr, n_tiles);
  return MZGPU_OK;
}

int32_t mz_topk_explode(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const TopKOrder& to, u64* d_arr,
                        u64* d_errs, u64* d_cnt) {
  MZ_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, 16, ctx->stream));
  if (n_ub == 0) return MZGPU_OK;
  const unsigned grid = grid_of(ctx, (n_ub + RT - 1) / RT);
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * (to.in_words * 8 + TK_NW * 8) : 0);
  MZ_LAUNCH(ctx, k_topk_explode, grid, RT, 0, d_rows, n, to, d_arr, d_errs, (unsigned long long*)d_cnt);
  return MZGPU_OK;
}

int32_t mz_topk_window_async(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const TraceView& prior,
                             const TopKOrder& to, u64* d_win, u64* d_out, u64 out_cap, u64* d_out_len) {
  LookBack lb;
  unsigned grid;
  MZ_TRY(lb_launch_setup(ctx, n, n_ub, 2 * TK_NW * 8, &lb, &grid));
  return mz_dispatch<InRowWords>(ctx, (int)to.in_words, "topk window", [&](auto IW) {
    MZ_LAUNCH(ctx, k_topk_window_lb<IW>, grid, RT, 0, d_rows, n, prior, to.limit, lb, d_win, d_out,
              out_cap, d_out_len, ctx->d_status);
    return MZGPU_OK;
  });
}

int32_t mz_topk_window(mzgpu_ctx* ctx, const u64* d_rows, u64 n, const TraceView& prior, const TopKOrder& to,
                       DevMem* win, DevMem* out, u64* n_out) {
  *n_out = 0;
  if (n == 0) return MZGPU_OK;
  auto count = [&](u32* tile_counts, u64 n_tiles) {
    return mz_dispatch<InRowWords>(ctx, (int)to.in_words, "topk window", [&](auto IW) {
      MZ_LAUNCH(ctx, (k_topk_window<IW, false>), (unsigned)n_tiles, RT, 0, d_rows, n, prior, to.limit, tile_counts,
                (const u32*)nullptr, (u64*)nullptr, (u64*)nullptr);
      return MZGPU_OK;
    });
  };
  auto alloc = [&](u64 total) {
    if (total == 0) return MZGPU_OK;  // (no window change: the outputs stay unallocated)
    MZ_TRY(win->alloc(ctx, total * TK_NW * 8));
    return out->alloc(ctx, total * to.in_words * 8);
  };
  auto write = [&](const u32* tile_base, u64 n_tiles) {
    return mz_dispatch<InRowWords>(ctx, (int)to.in_words, "topk window", [&](auto IW) {
      MZ_LAUNCH(ctx, (k_topk_window<IW, true>), (unsigned)n_tiles, RT, 0, d_rows, n, prior, to.limit,
                (u32*)nullptr, tile_base, win->as<u64>(), out->as<u64>());
      return MZGPU_OK;
    });
  };
  return two_pass(ctx, n, n_out, count, alloc, write);
}

int32_t mz_topk_basic_explode(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const TopKOrder& to, u64* d_arr) {
  if (n_ub == 0) return MZGPU_OK;
  const unsigned grid = grid_of(ctx, (n_ub + RT - 1) / RT);
  MZ_BYTES(ctx, n.p == nullptr ? n.imm * (to.in_words * 8 + TK_NW * 8) : 0);
  MZ_LAUNCH(ctx, k_topk_basic_explode, grid, RT, 0, d_rows, n, to, d_arr);
  return MZGPU_OK;
}

int32_t mz_topk_basic_async(mzgpu_ctx* ctx, const u64* d_rows, DLen n, u64 n_ub, const TraceView& prior,
                            const TraceView& negs_tv, const TopKOrder& to, i64 offset, u64* d_out, u64 out_cap,
                            u64* d_out_len, u64* d_errs, u64* d_negs, u64 side_cap, u64* d_side_len) {
  MZ_CUDA(ctx, cudaMemsetAsync(d_side_len, 0, 16, ctx->stream));
  LookBack lb;
  unsigned grid;
  MZ_TRY(lb_launch_setup(ctx, n, n_ub, 2 * TK_NW * 8 + 2 * to.in_words * 8, &lb, &grid));
  return mz_dispatch<InRowWords>(ctx, (int)to.in_words, "topk basic", [&](auto IW) {
    MZ_LAUNCH(ctx, k_topk_basic_lb<IW>, grid, RT, 0, d_rows, n, prior, negs_tv, to.limit, offset, lb, d_out, out_cap,
              d_out_len, d_errs, d_negs, side_cap, (unsigned long long*)d_side_len, ctx->d_status);
    return MZGPU_OK;
  });
}

int32_t mz_topk_basic(mzgpu_ctx* ctx, const u64* d_rows, u64 n, const TraceView& prior, const TraceView& negs_tv,
                      const TopKOrder& to, i64 offset, DevMem* out, u64* n_out, u64* d_errs, u64* d_negs,
                      u64 side_cap, u64* d_side_len) {
  *n_out = 0;
  MZ_CUDA(ctx, cudaMemsetAsync(d_side_len, 0, 16, ctx->stream));
  if (n == 0) return MZGPU_OK;
  auto count = [&](u32* tile_counts, u64 n_tiles) {
    return mz_dispatch<InRowWords>(ctx, (int)to.in_words, "topk basic", [&](auto IW) {
      MZ_LAUNCH(ctx, (k_topk_basic<IW, false>), (unsigned)n_tiles, RT, 0, d_rows, n, prior, negs_tv, to.limit, offset,
                tile_counts, (const u32*)nullptr, (u64*)nullptr, (u64*)nullptr, (u64*)nullptr, (u64)0,
                (unsigned long long*)nullptr, ctx->d_status);
      return MZGPU_OK;
    });
  };
  auto alloc = [&](u64 total) { return out->alloc(ctx, std::max<u64>(total, 1) * to.in_words * 8); };
  auto write = [&](const u32* tile_base, u64 n_tiles) {
    return mz_dispatch<InRowWords>(ctx, (int)to.in_words, "topk basic", [&](auto IW) {
      MZ_LAUNCH(ctx, (k_topk_basic<IW, true>), (unsigned)n_tiles, RT, 0, d_rows, n, prior, negs_tv, to.limit, offset,
                (u32*)nullptr, tile_base, out->as<u64>(), d_errs, d_negs, side_cap, (unsigned long long*)d_side_len,
                ctx->d_status);
      return MZGPU_OK;
    });
  };
  const u64 n_tiles = (n + RT - 1) / RT;
  MZ_TRY(two_pass(ctx, n, n_out, count, alloc, write));
  // a batch whose keys change no window can still change their negative counts and error states
  if (*n_out == 0) return write(nullptr, n_tiles);
  return MZGPU_OK;
}
