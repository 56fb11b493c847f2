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
inline uint32_t lookup_depth(uint64_t m, uint64_t n, uint64_t data_len, uint64_t frame_bytes, uint64_t budget) {
    if (n < 2 || m == 0) return 0;
    uint32_t dmax = 0;
    while (dmax < kLookupMaxDepth && (2ull << dmax) <= n) dmax++;
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

} // namespace dbeel
