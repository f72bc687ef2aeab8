// oracle/mzo_batch.hpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// CPU restatement of the merge batcher (chunker, chain policy, 2-way chain
// merge, extract), the OrdVal batch (CSR), its cursor and the batch merger.
//
// Sources followed (under /root/reference):
//   chunker   src/timely-util/src/columnation.rs:442-546 (ColumnationChunker)
//   merge     src/timely-util/src/columnation.rs:579-634 (InternalMerge::merge_from)
//             + differential-dataflow 0.23.0 merge_batcher::InternalMerger::merge
//               (external crate; control flow mirrored by the in-tree
//               src/timely-util/src/columnar/batcher.rs:635-753)
//   extract   src/timely-util/src/columnation.rs:636-655
//   batcher   differential-dataflow 0.23.0 MergeBatcher::{push_container,
//             insert_chain, seal} (external; protocol visible at
//             src/timely-util/src/operator.rs:583-633)
//   batch     OrdValBatch field layout src/compute/src/extensions/arrange.rs:325-330,
//             counts src/timely-util/src/columnation.rs:406-429
//   merger    differential-dataflow 0.23.0 ord_neu OrdValMerger semantics
//             (SURVEY.md Appendix A4)
// Parity pin: golden vectors batcher.rs:1016-1093 and the proptest properties
// :1185-1333 are reproduced in tests/test_oracle_golden.py.
#pragma once
#include <cassert>
#include <memory>

#include "mzo_rows.hpp"

namespace mzo {

static const u64 FRONTIER_EMPTY = MZGPU_FRONTIER_EMPTY;

// upper.less_equal(time) for a 0/1-element antichain of u64.
static inline bool frontier_less_equal(u64 upper, u64 time) {
  return upper != FRONTIER_EMPTY && upper <= time;
}

// ------------------------------------------------------------- chunks
template <class R>
struct Chunk {
  std::vector<R> rows;
};

template <class R>
static inline size_t chunk_capacity() {
  // ColumnationChunker::chunk_capacity with BUFFER_SIZE_BYTES = 64 KiB
  // (columnation.rs:464-474).
  return (64u << 10) / sizeof(R);
}

template <class R>
using Chain = std::vector<Chunk<R>>;

template <class R>
size_t chain_rows(const Chain<R>& c) {
  size_t n = 0;
  for (auto& ch : c) n += ch.rows.size();
  return n;
}

// InternalMerge::merge_from, 2-input and 1-input forms (columnation.rs:579-634).
template <class R>
void merge_from2(Chunk<R>& self, const Chunk<R>& o1, const Chunk<R>& o2, size_t* p) {
  const size_t cap = chunk_capacity<R>();
  while (p[0] < o1.rows.size() && p[1] < o2.rows.size() && self.rows.size() < cap) {
    const R& a = o1.rows[p[0]];
    const R& b = o2.rows[p[1]];
    if (Tr<R>::less(a, b)) {
      self.rows.push_back(a);
      p[0]++;
    } else if (Tr<R>::less(b, a)) {
      self.rows.push_back(b);
      p[1]++;
    } else {
      R s = a;
      Tr<R>::add(s, b);
      if (!Tr<R>::zero(s)) self.rows.push_back(s);
      p[0]++;
      p[1]++;
    }
  }
}

template <class R>
void merge_from1(Chunk<R>& self, Chunk<R>& other, size_t* pos) {
  if (self.rows.empty() && *pos == 0) {
    std::swap(self.rows, other.rows);
    return;
  }
  for (size_t i = *pos; i < other.rows.size(); ++i) self.rows.push_back(other.rows[i]);
  *pos = other.rows.size();
}

// InternalMerger::merge over two chains.
template <class R>
void merge_chains(Chain<R>&& list1, Chain<R>&& list2, Chain<R>& output) {
  const size_t cap = chunk_capacity<R>();
  size_t i1 = 0, i2 = 0;
  Chunk<R> heads[2];
  if (i1 < list1.size()) heads[0] = std::move(list1[i1++]);
  if (i2 < list2.size()) heads[1] = std::move(list2[i2++]);
  size_t pos[2] = {0, 0};
  Chunk<R> result;
  while (pos[0] < heads[0].rows.size() && pos[1] < heads[1].rows.size()) {
    merge_from2(result, heads[0], heads[1], pos);
    if (pos[0] >= heads[0].rows.size()) {
      heads[0] = i1 < list1.size() ? std::move(list1[i1++]) : Chunk<R>();
      pos[0] = 0;
    }
    if (pos[1] >= heads[1].rows.size()) {
      heads[1] = i2 < list2.size() ? std::move(list2[i2++]) : Chunk<R>();
      pos[1] = 0;
    }
    if (result.rows.size() >= cap) {
      output.push_back(std::move(result));
      result = Chunk<R>();
    }
  }
  // drain_side for each input: copy the partial head, then hand remaining
  // whole chunks over without per-element copies.
  for (int side = 0; side < 2; ++side) {
    Chain<R>& list = side == 0 ? list1 : list2;
    size_t& li = side == 0 ? i1 : i2;
    if (pos[side] < heads[side].rows.size()) merge_from1(result, heads[side], &pos[side]);
    if (!result.rows.empty()) {
      output.push_back(std::move(result));
      result = Chunk<R>();
    }
    while (li < list.size()) output.push_back(std::move(list[li++]));
    heads[side] = Chunk<R>();
    pos[side] = 0;
  }
}

// Merger::extract over a merged chain (columnation.rs:636-655 driven by
// InternalMerger::extract): ship = !upper.less_equal(t), keep otherwise;
// frontier = antichain (min) of kept times.
template <class R>
void extract_chain(Chain<R>&& merged, u64 upper, u64* frontier, Chain<R>& ship, Chain<R>& kept) {
  const size_t cap = chunk_capacity<R>();
  Chunk<R> keep, ready;
  for (auto& buffer : merged) {
    for (const R& r : buffer.rows) {
      u64 t = Tr<R>::time(r);
      if (frontier_less_equal(upper, t)) {
        if (*frontier == FRONTIER_EMPTY || t < *frontier) *frontier = t;
        keep.rows.push_back(r);
      } else {
        ready.rows.push_back(r);
      }
      if (keep.rows.size() >= cap) {
        kept.push_back(std::move(keep));
        keep = Chunk<R>();
      }
      if (ready.rows.size() >= cap) {
        ship.push_back(std::move(ready));
        ready = Chunk<R>();
      }
    }
  }
  if (!keep.rows.empty()) kept.push_back(std::move(keep));
  if (!ready.rows.empty()) ship.push_back(std::move(ready));
}

// ------------------------------------------------------------- batches
struct Desc {
  u64 lower = 0, upper = 0, since = 0;
};

// Generic immutable batch of sorted, consolidated rows + the CSR index arrays
// of OrdValBatch (`keys`, `vals.offs`, `upds.offs`).  For rows without a val
// (RACC, ROUT) `val_offs` indexes updates per key-run of equal non-time data.
template <class R>
struct Batch {
  std::vector<R> rows;       // logically ((key,val),time,diff) in cursor order
  std::vector<u64> keys;     // distinct keys
  std::vector<u64> key_offs; // keys.size()+1 offsets into vals (val-run index)
  std::vector<u64> val_offs; // #val-runs+1 offsets into rows
  Desc desc;
  size_t len() const { return rows.size(); }
  bool is_empty() const { return rows.empty(); }
};

template <class R>
static inline bool same_data(const R& a, const R& b);
template <>
inline bool same_data<mzgpu_r32>(const mzgpu_r32& a, const mzgpu_r32& b) {
  return a.key == b.key && a.val == b.val;
}
template <>
inline bool same_data<mzgpu_racc>(const mzgpu_racc& a, const mzgpu_racc& b) {
  return a.key == b.key;
}
template <>
inline bool same_data<mzgpu_rout>(const mzgpu_rout& a, const mzgpu_rout& b) {
  return a.key == b.key && a.count == b.count && a.sum_lo == b.sum_lo && a.sum_hi == b.sum_hi &&
         a.flags == b.flags;
}

// OrdValBuilder::{with_capacity,push,done} (external; SURVEY.md A3): consume
// sorted consolidated chunks, emit CSR.
template <class R>
std::shared_ptr<Batch<R>> build_batch(Chain<R>& chain, Desc desc) {
  auto b = std::make_shared<Batch<R>>();
  b->desc = desc;
  b->rows.reserve(chain_rows(chain));
  for (auto& ch : chain)
    for (auto& r : ch.rows) b->rows.push_back(r);
  chain.clear();
  const auto& rows = b->rows;
  b->key_offs.push_back(0);
  b->val_offs.push_back(0);
  for (size_t i = 0; i < rows.size(); ++i) {
    bool new_key = i == 0 || rows[i].key != rows[i - 1].key;
    bool new_val = new_key || !same_data(rows[i], rows[i - 1]);
    if (new_val && i != 0) b->val_offs.push_back(i);
    if (new_key) {
      if (i != 0) b->key_offs.push_back(b->val_offs.size() - 1);
      b->keys.push_back(rows[i].key);
    }
  }
  if (!rows.empty()) {
    b->val_offs.push_back(rows.size());
    b->key_offs.push_back(b->val_offs.size() - 1);
  }
  return b;
}

template <class R>
std::shared_ptr<Batch<R>> build_batch_from_rows(std::vector<R> rows, Desc desc) {
  consolidate(rows);
  Chain<R> chain;
  Chunk<R> c;
  c.rows = std::move(rows);
  chain.push_back(std::move(c));
  return build_batch(chain, desc);
}

template <class R>
std::shared_ptr<Batch<R>> empty_batch(u64 lower, u64 upper, u64 since) {
  Chain<R> chain;
  Desc d;
  d.lower = lower;
  d.upper = upper;
  d.since = since;
  return build_batch(chain, d);
}

// ------------------------------------------------------------- batcher
// MergeBatcher<Vec<..>, ColumnationChunker<..>, ColInternalMerger<..>>
// (src/compute/src/typedefs.rs:121-126).
template <class R>
struct Batcher {
  std::vector<R> pending;            // ColumnationChunker::pending
  std::vector<Chain<R>> chains;      // MergeBatcher::chains
  u64 lower = 0;                     // MergeBatcher::lower
  u64 frontier = FRONTIER_EMPTY;     // MergeBatcher::frontier

  // ColumnationChunker::form_chunk (columnation.rs:477-488).
  void form_chunk(std::vector<Chunk<R>>& ready) {
    const size_t cap = chunk_capacity<R>();
    consolidate(pending);
    if (pending.size() >= cap) {
      size_t off = 0;
      while (pending.size() - off > cap) {
        Chunk<R> c;
        c.rows.assign(pending.begin() + off, pending.begin() + off + cap);
        ready.push_back(std::move(c));
        off += cap;
      }
      pending.erase(pending.begin(), pending.begin() + off);
    }
  }

  void insert_chain(Chain<R>&& chain) {
    if (chain.empty()) return;
    chains.push_back(std::move(chain));
    while (chains.size() > 1 &&
           chains[chains.size() - 1].size() >= chains[chains.size() - 2].size() / 2) {
      Chain<R> l1 = std::move(chains.back());
      chains.pop_back();
      Chain<R> l2 = std::move(chains.back());
      chains.pop_back();
      Chain<R> merged;
      merge_chains(std::move(l1), std::move(l2), merged);
      chains.push_back(std::move(merged));
    }
  }

  // Batcher::push_container: chunker.push_into + insert_chain per ready chunk
  // (columnation.rs:510-526).
  void push_container(const R* rows, size_t n) {
    const size_t cap2 = chunk_capacity<R>() * 2;
    size_t i = 0;
    std::vector<Chunk<R>> ready;
    while (i < n) {
      size_t take = std::min(n - i, cap2 - pending.size());
      pending.insert(pending.end(), rows + i, rows + i + take);
      i += take;
      if (pending.size() == cap2) form_chunk(ready);
    }
    for (auto& c : ready) {
      Chain<R> ch;
      ch.push_back(std::move(c));
      insert_chain(std::move(ch));
    }
  }

  size_t len() const {
    size_t n = pending.size();
    for (auto& c : chains) n += chain_rows(c);
    return n;
  }

  // Batcher::seal::<Builder>(upper).
  std::shared_ptr<Batch<R>> seal(u64 upper) {
    // chunker.finish() (columnation.rs:530-546)
    const size_t cap = chunk_capacity<R>();
    consolidate(pending);
    size_t off = 0;
    while (off < pending.size()) {
      size_t take = std::min(pending.size() - off, cap);
      Chunk<R> c;
      c.rows.assign(pending.begin() + off, pending.begin() + off + take);
      off += take;
      Chain<R> ch;
      ch.push_back(std::move(c));
      insert_chain(std::move(ch));
    }
    pending.clear();
    while (chains.size() > 1) {
      Chain<R> l1 = std::move(chains.back());
      chains.pop_back();
      Chain<R> l2 = std::move(chains.back());
      chains.pop_back();
      Chain<R> merged;
      merge_chains(std::move(l1), std::move(l2), merged);
      chains.push_back(std::move(merged));
    }
    Chain<R> merged;
    if (!chains.empty()) {
      merged = std::move(chains.back());
      chains.pop_back();
    }
    Chain<R> kept, readied;
    frontier = FRONTIER_EMPTY;
    extract_chain(std::move(merged), upper, &frontier, readied, kept);
    if (!kept.empty()) chains.push_back(std::move(kept));
    Desc d;
    d.lower = lower;
    d.upper = upper;
    d.since = 0;
    auto b = build_batch(readied, d);
    lower = upper;
    return b;
  }
};

// ------------------------------------------------------------- cursor
// Cursor::{get_key,seek_key,step_key,get_val,step_val,map_times} on a batch
// (usage: src/compute/src/render/join/mz_join_core.rs:606-621,816-837).
template <class R>
struct BatchCursor {
  const Batch<R>* b = nullptr;
  size_t key_idx = 0;
  size_t val_idx = 0;  // absolute index into val runs
  explicit BatchCursor(const Batch<R>* batch) : b(batch) { rewind_vals(); }
  bool key_valid() const { return key_idx < b->keys.size(); }
  u64 key() const { return b->keys[key_idx]; }
  void rewind_vals() {
    if (key_valid()) val_idx = b->key_offs[key_idx];
  }
  void step_key() {
    ++key_idx;
    rewind_vals();
  }
  // exponential + binary search forward (ord_neu seek via `advance`)
  void seek_key(u64 k) {
    size_t lo = key_idx, n = b->keys.size();
    if (lo < n && b->keys[lo] < k) {
      size_t step = 1;
      while (lo + step < n && b->keys[lo + step] < k) {
        lo += step;
        step <<= 1;
      }
      step >>= 1;
      while (step > 0) {
        if (lo + step < n && b->keys[lo + step] < k) lo += step;
        step >>= 1;
      }
      lo += 1;
    }
    key_idx = lo;
    rewind_vals();
  }
  bool val_valid() const { return key_valid() && val_idx < b->key_offs[key_idx + 1]; }
  const R& val_row() const { return b->rows[b->val_offs[val_idx]]; }
  void step_val() { ++val_idx; }
  template <class F>
  void map_times(F f) const {
    for (u64 u = b->val_offs[val_idx]; u < b->val_offs[val_idx + 1]; ++u) f(b->rows[u]);
  }
};

// CursorList: k-way merged cursor over the batches of a trace (external DD
// trace::cursor::CursorList; semantics per SURVEY.md a8).
template <class R>
struct CursorList {
  std::vector<BatchCursor<R>> cursors;
  std::vector<size_t> min_key;  // indices of cursors at the minimum key
  std::vector<size_t> min_val;  // among those, indices at the minimum val
  explicit CursorList(const std::vector<std::shared_ptr<Batch<R>>>& batches) {
    for (auto& b : batches) cursors.emplace_back(b.get());
    minimize_keys();
  }
  void minimize_keys() {
    min_key.clear();
    bool have = false;
    u64 mk = 0;
    for (size_t i = 0; i < cursors.size(); ++i) {
      if (!cursors[i].key_valid()) continue;
      u64 k = cursors[i].key();
      if (!have || k < mk) {
        have = true;
        mk = k;
        min_key.clear();
      }
      if (k == mk) min_key.push_back(i);
    }
    minimize_vals();
  }
  static bool val_less(const R& a, const R& b);
  void minimize_vals() {
    min_val.clear();
    const R* mv = nullptr;
    for (size_t i : min_key) {
      if (!cursors[i].val_valid()) continue;
      const R& v = cursors[i].val_row();
      if (mv == nullptr || data_less(v, *mv)) {
        mv = &v;
        min_val.clear();
      }
      if (same_data(v, *mv)) min_val.push_back(i);
    }
  }
  static bool data_less(const R& a, const R& b) {
    R x = a, y = b;
    Tr<R>::set_time(x, 0);
    Tr<R>::set_time(y, 0);
    return Tr<R>::less(x, y);
  }
  bool key_valid() const { return !min_key.empty(); }
  u64 key() const { return cursors[min_key[0]].key(); }
  void step_key() {
    for (size_t i : min_key) cursors[i].step_key();
    minimize_keys();
  }
  void seek_key(u64 k) {
    for (auto& c : cursors) c.seek_key(k);
    minimize_keys();
  }
  bool val_valid() const { return !min_val.empty(); }
  const R& val_row() const { return cursors[min_val[0]].val_row(); }
  void step_val() {
    for (size_t i : min_val) cursors[i].step_val();
    minimize_vals();
  }
  template <class F>
  void map_times(F f) const {
    for (size_t i : min_val) cursors[i].map_times(f);
  }
};

// ------------------------------------------------------ batch merger (a7)
// Batch::Merger for OrdValBatch: merge keys -> vals -> (time,diff) lists with
// time.advance_by(since) (= max for totally ordered u64 times,
// src/repr/src/timestamp.rs:486-495; advance_by of the empty antichain leaves a time
// alone), consolidate each (key,val) history, drop empty vals and keys.  `b1.upper == b2.lower`.
template <class R>
std::shared_ptr<Batch<R>> merge_batches(const Batch<R>& b1, const Batch<R>& b2, u64 since) {
  std::vector<R> out;
  out.reserve(b1.rows.size() + b2.rows.size());
  std::vector<std::shared_ptr<Batch<R>>> none;
  BatchCursor<R> c1(&b1), c2(&b2);
  std::vector<R> hist;
  auto flush_val = [&](BatchCursor<R>* a, BatchCursor<R>* b) {
    hist.clear();
    auto push = [&](const R& r) {
      R x = r;
      if (since != FRONTIER_EMPTY && Tr<R>::time(x) < since) Tr<R>::set_time(x, since);
      hist.push_back(x);
    };
    if (a) a->map_times(push);
    if (b) b->map_times(push);
    consolidate(hist);
    for (auto& r : hist) out.push_back(r);
  };
  auto copy_key = [&](BatchCursor<R>& c) {
    while (c.val_valid()) {
      flush_val(&c, nullptr);
      c.step_val();
    }
  };
  while (c1.key_valid() && c2.key_valid()) {
    if (c1.key() < c2.key()) {
      copy_key(c1);
      c1.step_key();
    } else if (c2.key() < c1.key()) {
      copy_key(c2);
      c2.step_key();
    } else {
      while (c1.val_valid() && c2.val_valid()) {
        const R& v1 = c1.val_row();
        const R& v2 = c2.val_row();
        if (same_data(v1, v2)) {
          flush_val(&c1, &c2);
          c1.step_val();
          c2.step_val();
        } else if (CursorList<R>::data_less(v1, v2)) {
          flush_val(&c1, nullptr);
          c1.step_val();
        } else {
          flush_val(&c2, nullptr);
          c2.step_val();
        }
      }
      copy_key(c1);
      copy_key(c2);
      c1.step_key();
      c2.step_key();
    }
  }
  while (c1.key_valid()) {
    copy_key(c1);
    c1.step_key();
  }
  while (c2.key_valid()) {
    copy_key(c2);
    c2.step_key();
  }
  Chain<R> chain;
  Chunk<R> ch;
  ch.rows = std::move(out);
  chain.push_back(std::move(ch));
  Desc d;
  d.lower = b1.desc.lower;
  d.upper = b2.desc.upper;
  d.since = since;
  return build_batch(chain, d);
}

}  // namespace mzo
