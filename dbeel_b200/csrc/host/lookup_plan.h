// lookup_plan.h -- the read plan of a batched read from SSTable files (dbeel_get_values_stream).  Plain C++ with the search
// step marked for both sides: the kernels (lookup_stream.cuh) run the same step, and the planner is tested on a box without a
// GPU (tests/lookup_plan_test.cc).
//
// Both search modes of lookup.cuh are deterministic probe trees over .index positions: the next probe depends only on the
// comparisons so far.  Number the nodes as a heap (root 1; the child after Ordering::Greater is 2k, after Less 2k + 1).  A
// search that is still open after D probes sits at node 2^D + leaf, and every probe it can still make lies in that leaf's
// interval of index records.  So a batch reads the top D levels of the tree ("fences": an index record and its key frame per
// node) and the intervals its queries reach, and nothing else.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "page_cache.h"

#ifdef __CUDACC__
#define DBEEL_HD __host__ __device__ __forceinline__
#else
#define DBEEL_HD inline
#endif

namespace dbeel {

// One search inside one table.  Reference mode: a = low, b = high, half; exact mode: a = lo, b = hi.
struct SearchState {
    uint64_t a, b, half;
    uint32_t done, pad;
};

DBEEL_HD SearchState search_init(uint32_t mode, uint64_t n) {
    SearchState s;
    if (mode == 0) { s.a = 0; s.b = n ? n - 1 : 0; s.half = n / 2; s.done = n == 0; }
    else { s.a = 0; s.b = n; s.half = 0; s.done = n == 0; }
    s.pad = 0;
    return s;
}

// the record the next probe reads
DBEEL_HD uint64_t search_pos(uint32_t mode, const SearchState &s) { return mode == 0 ? s.half : s.a + (s.b - s.a) / 2; }

// After a probe that compared c != 0 and was not bad: exactly the updates of lookup_query's loops (lookup.cuh).
DBEEL_HD void search_step(uint32_t mode, uint64_t n, SearchState *s, int c) {
    if (mode == 0) {
        const uint64_t half = s->half;
        s->a = c < 0 ? half + 1 : s->a;                          // Ordering::Less
        s->b = c > 0 ? (half > 1 ? half : 1) - 1 : s->b;         // Ordering::Greater: max(half, 1) - 1
        bool done = half == 0 || half == n;
        s->half = (s->b + s->a) / 2;
        s->done = done || s->a > s->b;
    } else {
        const uint64_t mid = s->a + (s->b - s->a) / 2;
        if (c < 0) s->a = mid + 1; else s->b = mid;
        s->done = s->a >= s->b;
    }
}

// the records [*lo, *hi) every later probe of an open search lies in
DBEEL_HD void search_interval(uint32_t mode, const SearchState &s, uint64_t *lo, uint64_t *hi) {
    *lo = s.a;
    *hi = mode == 0 ? s.b + 1 : s.b;
}

constexpr uint32_t kLookupMaxDepth = 16;       // at most 2^16 leaves, 2^16 - 1 fences
constexpr uint64_t kLookupFenceCost = 4096;    // one small read, in bytes of a sequential one
constexpr uint64_t kLookupMergeGap = 1024;     // .index reads closer than this become one (.data reads merge when they touch)

// The top `depth` levels of the probe tree of a table of n records: state[k] for every node k < 2^(depth + 1), open[k] = the
// search is still open on arriving at k (internal nodes: k is probed; leaves: k is resumed).
struct ProbeTree {
    uint32_t mode = 0, depth = 0;
    uint64_t n = 0;
    std::vector<SearchState> state;
    std::vector<uint8_t> open;
};

inline void plan_probe_tree(uint32_t mode, uint64_t n, uint32_t depth, ProbeTree *t) {
    t->mode = mode;
    t->depth = depth;
    t->n = n;
    const uint64_t nodes = 2ull << depth;
    t->state.assign(nodes, SearchState{});
    t->open.assign(nodes, 0);
    t->state[1] = search_init(mode, n);
    t->open[1] = !t->state[1].done;
    for (uint64_t k = 1; k < (1ull << depth); k++) {
        if (!t->open[k]) continue;
        for (int right = 0; right < 2; right++) {
            SearchState c = t->state[k];
            search_step(mode, n, &c, right ? -1 : 1);
            t->state[2 * k + right] = c;
            t->open[2 * k + right] = !c.done;
        }
    }
}

// The fence depth for m queries on a table of n records and data_len bytes: about 2^D = sqrt(m * data_len / fence cost)
// balances the fence reads against m leaf windows of data_len / 2^D bytes; at least deep enough that a leaf is a quarter
// of the budget, never deeper than the tree (log2 n) or kLookupMaxDepth, and the fences (index record + key frame of up to
// frame_bytes each) stay within half the budget.
inline uint32_t lookup_max_depth(uint64_t n) { // floor(log2 n), at most kLookupMaxDepth
    uint32_t d = 0;
    while (d < kLookupMaxDepth && (2ull << d) <= n) d++;
    return d;
}

inline uint32_t lookup_depth(uint64_t m, uint64_t n, uint64_t data_len, uint64_t frame_bytes, uint64_t budget) {
    if (n < 2 || m == 0) return 0;
    const uint32_t dmax = lookup_max_depth(n);
    const double want = 0.5 * std::log2(std::max(1.0, (double)m * (double)data_len / (double)kLookupFenceCost));
    uint32_t d = (uint32_t)std::min<double>(dmax, std::ceil(want));
    while (d < dmax && (data_len >> d) > budget / 4) d++;
    while (d > 0 && (1ull << d) * (16 + frame_bytes + 32) > budget / 2) d--;
    return d;
}

struct ByteRange {
    uint64_t lo, hi;
};

// Sorted by lo; ranges that overlap or lie closer than `gap` become one.
inline std::vector<ByteRange> merge_ranges(std::vector<ByteRange> r, uint64_t gap) {
    std::sort(r.begin(), r.end(), [](const ByteRange &x, const ByteRange &y) { return x.lo < y.lo || (x.lo == y.lo && x.hi < y.hi); });
    std::vector<ByteRange> out;
    for (const ByteRange &x : r) {
        if (!out.empty() && x.lo <= out.back().hi + gap) out.back().hi = std::max(out.back().hi, x.hi);
        else out.push_back(x);
    }
    return out;
}

inline uint64_t rd_le(const uint8_t *p, int nb) {
    uint64_t v = 0;
    for (int b = nb - 1; b >= 0; b--) v = (v << 8) | p[b];
    return v;
}

// The .data bytes a probe of index record `ix` (16 bytes) can touch, for query keys of at most max_klen bytes: the u64
// length prefix and up to max_klen key bytes, cut at the end of .data; empty when the record points past the file (the
// probe reports it corrupt without reading).  Computed from the record alone, so an index that lies about key_size cannot
// move a key frame outside its window; the prefix is checked against data_len by the probe itself.
inline bool probe_frame(const uint8_t *ix, uint64_t data_len, uint64_t max_klen, ByteRange *out) {
    const uint64_t off = rd_le(ix, 8);
    if (off > data_len || data_len - off < 8) return false;
    const uint64_t avail = data_len - off;
    out->lo = off;
    out->hi = off + std::min<uint64_t>(avail, 8 + max_klen);
    return true;
}

// The bytes of a leaf record the search and a hit's copy can touch: its probe frame and, when the record could answer a
// query of at most max_klen bytes (8 <= key_size <= 8 + max_klen, full_size >= key_size + 24, the entry inside .data),
// its whole entry [off, off + full_size), which is copied out of the window when it answers.
inline bool record_window(const uint8_t *ix, uint64_t data_len, uint64_t max_klen, ByteRange *out) {
    if (!probe_frame(ix, data_len, max_klen, out)) return false;
    const uint64_t ks = rd_le(ix + 8, 4), fs = rd_le(ix + 12, 4);
    if (ks >= 8 && ks <= 8 + max_klen && fs >= ks + 24 && fs <= data_len - out->lo) out->hi = std::max(out->hi, out->lo + fs);
    return true;
}

// The window of a leaf: the union of the record windows of its index slice (count records), or false when none touches
// .data.  On files the writer produced this is exactly the leaf's records' byte range.
inline bool leaf_window(const uint8_t *slice, uint64_t count, uint64_t data_len, uint64_t max_klen, ByteRange *out) {
    bool any = false;
    for (uint64_t r = 0; r < count; r++) {
        ByteRange f;
        if (!record_window(slice + 16 * r, data_len, max_klen, &f)) continue;
        if (!any) { *out = f; any = true; }
        out->lo = std::min(out->lo, f.lo);
        out->hi = std::max(out->hi, f.hi);
    }
    return any;
}

// A leaf the fence descent touched: leaf `leaf` of table t of the batch, whose open searches resume in records [a, b).
struct TouchedLeaf {
    uint32_t t, leaf;
    uint64_t a, b;
};

// Appends the leaves L of pt (table t) with touched[L] set, ascending.
inline void touched_leaves(const ProbeTree &pt, uint32_t t, const uint8_t *touched, std::vector<TouchedLeaf> *out) {
    const uint64_t leaf0 = 1ull << pt.depth;
    for (uint64_t L = 0; L < leaf0; L++) {
        if (!touched[L]) continue;
        uint64_t a, b;
        search_interval(pt.mode, pt.state[leaf0 + L], &a, &b);
        out->push_back(TouchedLeaf{t, (uint32_t)L, a, b});
    }
}

// Cuts touched leaves, in the order they are loaded, into groups of about group_bytes.  A leaf costs its records at 16
// index bytes plus table t's mean entry (ceil(data_len[t] / n[t]), 0 for an empty table), and 8 + max_klen for a probe
// frame; with a page cache (paged), two more pages, as its slice and window each end in pages of their own.  A group
// holds at least one leaf.  Group g is leaves [cut[g], cut[g + 1]) of the returned cut.
inline uint64_t leaf_bytes(const TouchedLeaf &l, uint64_t n, uint64_t data_len, uint64_t max_klen, bool paged) {
    return (l.b - l.a) * (16 + (n ? (data_len + n - 1) / n : 0)) + 8 + max_klen + (paged ? 2 * kPageBytes : 0);
}

inline std::vector<size_t> group_leaves(const std::vector<TouchedLeaf> &leaves, const std::vector<uint64_t> &n,
                                        const std::vector<uint64_t> &data_len, uint64_t max_klen, uint64_t group_bytes, bool paged) {
    std::vector<size_t> cut = {0};
    uint64_t est = 0;
    for (size_t k = 0; k < leaves.size(); k++) {
        const TouchedLeaf &l = leaves[k];
        const uint64_t bytes = leaf_bytes(l, n[l.t], data_len[l.t], max_klen, paged);
        if (k > cut.back() && est + bytes > group_bytes) {
            cut.push_back(k);
            est = 0;
        }
        est += bytes;
    }
    if (!leaves.empty()) cut.push_back(leaves.size());
    return cut;
}

// ---- batched reads across readers (dbeel_readers_get_values): one level of many (batch, table) pairs
//
// Pair p of a level: its table's n and data_len, its batch's longest key, and the page cache its leaves go through
// (cache_bytes index, or -1 for none).  TouchedLeaf.t is the pair.
struct LeafPair {
    uint64_t n, data_len, max_klen;
    int32_t cache;
};

// Cuts the touched leaves of a level, ascending pair, into groups.  Pair p's leaves are first cut exactly as its solo call
// cuts them (group_leaves with the partition budget, or with min(budget, its cache's bytes) when paged): those units keep
// every read of the pair inside the reads of its solo call, as the .index slices of a unit merge across the same gaps.
// Whole units then fill groups in order while the group's estimate stays within `budget` and the leaves of each cache c
// within cache_bytes[c]; a group holds at least one unit.
inline std::vector<size_t> group_leaves(const std::vector<TouchedLeaf> &leaves, const std::vector<LeafPair> &pairs, uint64_t budget,
                                        const std::vector<uint64_t> &cache_bytes) {
    std::vector<size_t> cut = {0};
    uint64_t est = 0;
    std::vector<uint64_t> est_c(cache_bytes.size(), 0);
    for (size_t k0 = 0; k0 < leaves.size();) {
        const uint32_t p = leaves[k0].t;
        const LeafPair &lp = pairs[p];
        size_t k1 = k0;
        while (k1 < leaves.size() && leaves[k1].t == p) k1++;
        const bool paged = lp.cache >= 0;
        const std::vector<uint64_t> n1 = {lp.n}, dl1 = {lp.data_len};
        std::vector<TouchedLeaf> local(leaves.begin() + k0, leaves.begin() + k1);
        for (TouchedLeaf &l : local) l.t = 0;
        const std::vector<size_t> unit = group_leaves(local, n1, dl1, lp.max_klen,
                                                      paged ? std::min(budget, cache_bytes[lp.cache]) : budget, paged);
        for (size_t u = 0; u + 1 < unit.size(); u++) {
            uint64_t bytes = 0;
            for (size_t k = unit[u]; k < unit[u + 1]; k++) bytes += leaf_bytes(local[k], lp.n, lp.data_len, lp.max_klen, paged);
            const size_t at = k0 + unit[u];
            if (at > cut.back() && (est + bytes > budget || (paged && est_c[lp.cache] + bytes > cache_bytes[lp.cache]))) {
                cut.push_back(at);
                est = 0;
                std::fill(est_c.begin(), est_c.end(), 0);
            }
            est += bytes;
            if (paged) est_c[lp.cache] += bytes;
        }
        k0 = k1;
    }
    if (!leaves.empty()) cut.push_back(leaves.size());
    return cut;
}

// ---- range reads across readers (dbeel_readers_get_ranges): seek batches and query groups of many batches
//
// Units of bytes[k], in order, cut into groups: a group takes the next unit while its bytes stay within `budget` and, for a
// unit that goes through page cache cache[k] >= 0, the bytes of that cache's units within cache_bytes[cache[k]] (an empty
// `cache`: none does); a group holds at least one unit.  Group g is units [cut[g], cut[g + 1]).
inline std::vector<size_t> pack_in_order(const std::vector<uint64_t> &bytes, uint64_t budget, const std::vector<int32_t> &cache = {},
                                         const std::vector<uint64_t> &cache_bytes = {}) {
    std::vector<size_t> cut = {0};
    uint64_t est = 0;
    std::vector<uint64_t> est_c(cache_bytes.size(), 0);
    for (size_t k = 0; k < bytes.size(); k++) {
        const int32_t c = cache.empty() ? -1 : cache[k];
        if (k > cut.back() && (est + bytes[k] > budget || (c >= 0 && est_c[c] + bytes[k] > cache_bytes[c]))) {
            cut.push_back(k);
            est = 0;
            std::fill(est_c.begin(), est_c.end(), 0);
        }
        est += bytes[k];
        if (c >= 0) est_c[c] += bytes[k];
    }
    if (!bytes.empty()) cut.push_back(bytes.size());
    return cut;
}

// Units [k0, k1) of batch `batch`.
struct BatchSpan {
    uint32_t batch;
    size_t k0, k1;
};

// The units of many batches in groups: batch b's units (cost[b], in order) are first cut as its solo call cuts them
// (pack_in_order with the budget alone); those solo groups then fill groups whole, in batch order, while the budget and
// each page cache's capacity hold (batch b goes through cache[b], -1 = none).  So every group of one batch is one of its
// solo groups, and one batch is grouped exactly as its solo call groups it.
inline std::vector<std::vector<BatchSpan>> pack_batches(const std::vector<std::vector<uint64_t>> &cost, const std::vector<int32_t> &cache,
                                                        uint64_t budget, const std::vector<uint64_t> &cache_bytes) {
    std::vector<BatchSpan> solo;
    std::vector<uint64_t> bytes;
    std::vector<int32_t> uc;
    for (uint32_t b = 0; b < cost.size(); b++) {
        const std::vector<size_t> cut = pack_in_order(cost[b], budget);
        for (size_t g = 0; g + 1 < cut.size(); g++) {
            solo.push_back(BatchSpan{b, cut[g], cut[g + 1]});
            uint64_t x = 0;
            for (size_t k = cut[g]; k < cut[g + 1]; k++) x += cost[b][k];
            bytes.push_back(x);
            uc.push_back(cache[b]);
        }
    }
    const std::vector<size_t> cut = pack_in_order(bytes, budget, uc, cache_bytes);
    std::vector<std::vector<BatchSpan>> out;
    for (size_t g = 0; g + 1 < cut.size(); g++) out.emplace_back(solo.begin() + cut[g], solo.begin() + cut[g + 1]);
    return out;
}

// ---- readers (dbeel_reader_*): fences kept on the device across batches
//
// A reader keeps, per table and mode, the fences of the top D_t levels of the probe tree: for every node k < 2^D_t its
// index record fix[k] (16 bytes), its frame address ffr[k] (8 bytes) and a frame slot of kReaderFrameSlot bytes.  Node
// k's state depends only on k, the mode and n (plan_probe_tree), never on the batch, so the set is read once and serves
// every later batch.  A cached frame holds the length prefix and at most kReaderFrameCap key bytes: cmp_key_bytes reads no
// more than min(fence key length, query key length) key bytes, so for a query of at most kReaderFrameCap bytes the
// truncated frame gives the comparison the whole key gives.  The "corrupt" decision (ffr = 0) depends only on the record
// and the length prefix, so it is cached as is.
constexpr uint64_t kReaderFrameCap = 64;
constexpr uint64_t kReaderFrameSlot = (8 + kReaderFrameCap + 15) / 16 * 16;
constexpr uint64_t kReaderNodeBytes = 16 + 8 + kReaderFrameSlot; // one node of one mode
constexpr uint64_t kReaderFenceBytesDefault = 64ull << 20;

// device bytes of one table's fences at depth d in both modes
inline uint64_t reader_fence_bytes(uint32_t d) { return d ? (2 * kReaderNodeBytes) << d : 0; }

// D_t for tables of n[t] records and data_len[t] bytes.  fixed[t] >= 0 is a depth chosen before (a table a reader shares
// with another keeps its fences), counted against the budget.  The rest of fence_bytes (0 = kReaderFenceBytesDefault)
// goes one level at a time to the table whose leaves are largest, (data_len + 16 n) >> D, ties to the lower position,
// while its next level fits; no table goes deeper than lookup_max_depth(n).  So the tables' fences fit fence_bytes
// whenever the fixed ones do.
inline std::vector<uint32_t> reader_depths(const std::vector<uint64_t> &n, const std::vector<uint64_t> &data_len,
                                           const std::vector<int32_t> &fixed, uint64_t fence_bytes) {
    const size_t nt = n.size();
    uint64_t left = fence_bytes ? fence_bytes : kReaderFenceBytesDefault;
    std::vector<uint32_t> d(nt, 0);
    std::vector<size_t> open;
    for (size_t t = 0; t < nt; t++) {
        if (fixed[t] >= 0) {
            d[t] = (uint32_t)fixed[t];
            left -= std::min(left, reader_fence_bytes(d[t]));
        } else {
            open.push_back(t);
        }
    }
    auto leaf = [&](size_t t) { return (data_len[t] + 16 * n[t]) >> d[t]; };
    auto later = [&](size_t a, size_t b) { return leaf(a) < leaf(b) || (leaf(a) == leaf(b) && a > b); };
    std::make_heap(open.begin(), open.end(), later);
    while (!open.empty()) {
        std::pop_heap(open.begin(), open.end(), later);
        const size_t t = open.back();
        open.pop_back();
        const uint64_t step = reader_fence_bytes(d[t] + 1) - reader_fence_bytes(d[t]);
        if (d[t] >= lookup_max_depth(n[t]) || step > left) continue; // the budget only shrinks: it never fits later
        left -= step;
        d[t]++;
        open.push_back(t);
        std::push_heap(open.begin(), open.end(), later);
    }
    return d;
}

// A batch descends a table's cached fences when its longest key fits the cached frames and the depth it would read per
// call (lookup_depth) is at most D_t; it then descends all D_t levels (deeper fences cost nothing once cached and make
// the leaves smaller).  Otherwise that table's fences are read for this batch, as dbeel_get_values_stream reads them.
inline bool reader_uses_cache(uint64_t max_klen, uint32_t want_depth, uint32_t cached_depth) {
    return max_klen <= kReaderFrameCap && want_depth <= cached_depth;
}

} // namespace dbeel
