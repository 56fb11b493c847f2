// scan_plan.h -- the partition plan of a streamed scan (dbeel_scan_stream).  Plain C++: no CUDA in here, so the planner is
// tested on a box without a GPU (tests/scan_plan_test.cc).
//
// A scan reads records in iteration order (lsm_tree.rs:210-281): table 0's index records, then table 1's, ...  A partition
// is a contiguous range of that sequence and may span tables.  For every table it touches, the partition's input slot holds
// the table's index slice and ONE .data window [min offset, max offset + full_size) over those records -- offsets need not
// run (the scan reads each entry at its (offset, full_size)), so the window is computed from the records, never assumed.
//
// A partition is cut before the record that would make its windows or its output bound (sum of full_size + 16 per record,
// which covers the index slice too) pass the budget; a record larger than the budget gets a partition of its own.  Any index
// order gives a correct plan; files the writer produced (running offsets) give disjoint windows that tile .data.
//
// The index is read in pieces through the caller's read callback and only the plan rows are kept, so the planner's memory
// is O(partitions), not O(records).  Every stop the reference would PANIC on is visible in the index alone -- full_size == 0,
// bytes past the end of .data, a table with no index record -- so the plan ends there and no partition carries such a record.
//
// Spans (dbeel_reader_scan's key ranges): per table ascending, disjoint record intervals; only they are read and planned.
// The plan is then the plan of the tables cut down to their spans (each .index = its span records back to back, .data
// whole; a table with records but an empty span dropped), with record numbers mapped back: the partitions cut at the same
// records, and a slice that runs across a span boundary in the cut table becomes one slice per span, each with the window
// of its own records.  The budget is charged with the cut table's window, which covers them all.  One more cut keeps a
// partition at kScanPartMaxSlices slices (k_scan_classify's table limit); whole-table plans never reach it.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <functional>
#include <map>
#include <vector>

namespace dbeel {

struct ScanSlice {    // one table's part of a partition
    uint32_t table;
    uint64_t rec_lo, rec_hi; // index records [rec_lo, rec_hi) of the table
    uint64_t win_lo, win_hi; // .data bytes [win_lo, win_hi) that hold them
};

struct ScanPart {
    uint32_t first_slice, n_slices; // ScanPlan::slices[first_slice .. + n_slices), ascending tables
    uint64_t n_rec;                 // records in the partition
    uint64_t data_bound;            // sum of full_size: the partition's output .data can be no larger
};

struct ScanPlan {
    std::vector<ScanPart> parts;
    std::vector<ScanSlice> slices;
    int32_t panic_table = -1; // the first record the reference would panic on (-1: none); the plan ends right before it
    uint64_t panic_record = 0;
};

// read(table, offset, len, dst): bytes [offset, offset + len) of table's .index file; returns 0 or the caller's error code.
using ScanIndexRead = std::function<int(uint32_t, uint64_t, uint64_t, void *)>;

constexpr uint64_t kScanPlanPiece = 1ull << 20;          // .index bytes per read while planning
constexpr uint64_t kScanPartMaxRecords = 0xFFFFFFF0ull - 1; // the whole-buffer scan's record limit, per partition
constexpr uint32_t kScanPartMaxSlices = 1024;               // = kScanMaxTables

struct ScanSpan { // index records [lo, hi) of one table
    uint64_t lo, hi;
};

// observe(table, record, offset, full_size): called for every record planned, in plan order (plan_merge's sampling).
using ScanRecordObserver = std::function<void(uint32_t, uint64_t, uint64_t, uint32_t)>;

// spans: null = every table whole (dbeel_scan_stream's plan), else (*spans)[t] = table t's spans.
inline int plan_scan(const uint64_t *data_len, const uint64_t *index_len, uint32_t n_tables, uint64_t budget,
                     const ScanIndexRead &read, ScanPlan *plan, const std::vector<std::vector<ScanSpan>> *spans = nullptr,
                     const ScanRecordObserver *observe = nullptr) {
    plan->parts.clear();
    plan->slices.clear();
    plan->panic_table = -1;
    plan->panic_record = 0;
    std::vector<uint8_t> buf(kScanPlanPiece);
    bool open = false;        // a partition is being filled
    ScanPart part = {};
    ScanSlice run = {};       // the open partition's records of the current table: the cut table's slice (budget)
    bool run_open = false;
    ScanSlice sl = {};        // the open slice: contiguous records of one span
    bool slice_open = false;
    uint64_t closed_win = 0;  // windows of the open partition's earlier tables
    uint64_t out_bound = 0;   // sum of (full_size + 16) in the open partition
    auto close_slice = [&]() {
        if (!slice_open) return;
        plan->slices.push_back(sl);
        part.n_slices++;
        slice_open = false;
    };
    auto close_run = [&]() {
        close_slice();
        if (!run_open) return;
        closed_win += run.win_hi - run.win_lo;
        run_open = false;
    };
    auto close_part = [&]() {
        if (!open) return;
        close_run();
        plan->parts.push_back(part);
        open = false;
    };
    for (uint32_t t = 0; t < n_tables; t++) {
        const uint64_t n = index_len[t] / 16; // lsm_tree.rs:225: floor(len / 16) records
        if (n == 0) { // its first index read runs past EOF
            plan->panic_table = (int32_t)t;
            close_part();
            return 0;
        }
        const std::vector<ScanSpan> whole = {ScanSpan{0, n}};
        for (const ScanSpan &span : spans ? (*spans)[t] : whole) {
            const uint64_t s_hi = span.hi < n ? span.hi : n;
            for (uint64_t r0 = span.lo; r0 < s_hi; r0 += kScanPlanPiece / 16) {
                const uint64_t m = s_hi - r0 < kScanPlanPiece / 16 ? s_hi - r0 : kScanPlanPiece / 16;
                const int rc = read(t, 16 * r0, 16 * m, buf.data());
                if (rc) return rc;
                for (uint64_t k = 0; k < m; k++) {
                    const uint8_t *q = buf.data() + 16 * k;
                    const uint64_t r = r0 + k;
                    uint64_t off = 0;
                    uint32_t fs = 0;
                    for (int b = 7; b >= 0; b--) off = (off << 8) | q[b];
                    for (int b = 15; b >= 12; b--) fs = (fs << 8) | q[b];
                    if (fs == 0 || off > data_len[t] || fs > data_len[t] - off) { // cached_file_reader.rs:68,82
                        plan->panic_table = (int32_t)t;
                        plan->panic_record = r;
                        close_part();
                        return 0;
                    }
                    if (observe) (*observe)(t, r, off, fs);
                    const uint64_t lo = off, hi = off + fs;
                    const bool same = run_open && run.table == t;
                    const bool joins = slice_open && sl.table == t && sl.rec_hi == r; // extends the open slice
                    if (open) { // would this record push the partition past the budget?
                        const uint64_t w = same ? (hi > run.win_hi ? hi : run.win_hi) - (lo < run.win_lo ? lo : run.win_lo)
                                                : (run_open ? run.win_hi - run.win_lo : 0) + fs;
                        const uint32_t slices = part.n_slices + (slice_open ? 1u : 0u) + (joins ? 0u : 1u);
                        if (closed_win + w > budget || out_bound + fs + 16 > budget || part.n_rec + 1 > kScanPartMaxRecords ||
                            slices > kScanPartMaxSlices)
                            close_part();
                    }
                    if (!open) {
                        part = ScanPart{(uint32_t)plan->slices.size(), 0, 0, 0};
                        closed_win = 0;
                        out_bound = 0;
                        open = true;
                    }
                    if (run_open && run.table != t) close_run();
                    if (!run_open) {
                        run = ScanSlice{t, r, r, lo, hi};
                        run_open = true;
                    }
                    if (slice_open && (sl.table != t || sl.rec_hi != r)) close_slice();
                    if (!slice_open) {
                        sl = ScanSlice{t, r, r, lo, hi};
                        slice_open = true;
                    }
                    if (lo < run.win_lo) run.win_lo = lo;
                    if (hi > run.win_hi) run.win_hi = hi;
                    if (lo < sl.win_lo) sl.win_lo = lo;
                    if (hi > sl.win_hi) sl.win_hi = hi;
                    run.rec_hi = sl.rec_hi = r + 1;
                    part.n_rec++;
                    part.data_bound += fs;
                    out_bound += fs + 16;
                }
            }
        }
    }
    close_part();
    return 0;
}

// ---- plan_merge: key-aligned partitions (dbeel_reader_get_range).  Partition c is the key interval [cuts[c - 1], cuts[c])
// (open at both ends of the key space) and holds, for every table, the span records in that interval, so a destination's
// merged output is the concatenation of its partitions' merged outputs.  The plan is a ScanPlan, run by run_scan_plan.
//   1. plan_scan over the spans.  One partition (or a PANIC record in the spans): that plan, and nothing else is read.
//      The same pass samples every table's span records about budget / (2 * tables) bytes apart (full_size + 16 each), and
//      the first record of every span when there are more spans than a partition may hold slices.
//   2. The sampled keys (key()) sorted and deduplicated are the splitters; seek() finds each in every table.  A splitter
//      any table could not seek is dropped; cuts are clamped to be monotone per table, so the intervals tile the spans even
//      on a table whose keys do not ascend (the device stage reports that table).
//   3. A second pass over the span .index slices cuts each table's span records at its cuts (one piece per interval and
//      span, with its window and bytes), and adjacent intervals are merged greedily up to the budget by plan_scan's rules.
//      A slice's window never passes the sum of its records' full_size: a record whose entry lies outside that starts a
//      new slice, so windows are bounded by the bytes they hold whatever the offsets.
// On keys that ascend, an interval holds at most one sampling step of each table, so every partition is within the budget
// plus one record per table (MergePlan::refused otherwise: nothing is planned past that bound).  Memory is
// O(samples + pieces), never O(records).
struct MergePlan {
    ScanPlan plan;
    std::vector<std::vector<uint8_t>> cuts; // plan.parts.size() - 1 ascending splitter keys
    // A key interval does not fit one partition -- its bytes pass the budget plus one record per table, or it holds more
    // slices or records than a partition may: some table's span keys do not ascend, or a splitter was dropped.  The plan
    // is then empty.
    bool refused = false;
};

// key(table, offset, full_size, key, ok): the key of the entry at .data offset (*ok = false when it does not decode);
// returns 0 or the caller's error code.
using MergeKeyRead = std::function<int(uint32_t, uint64_t, uint32_t, std::vector<uint8_t> *, bool *)>;
// seek(keys, pos): pos[t * keys.size() + j] = the first record of table t whose key is >= keys[j] (seek_t of
// dbeel_reader_scan), ~0 when the search failed; returns 0 or an error code.
using MergeSeek = std::function<int(const std::vector<std::vector<uint8_t>> &, std::vector<uint64_t> *)>;

inline int plan_merge(const uint64_t *data_len, const uint64_t *index_len, uint32_t n_tables, uint64_t budget,
                      const std::vector<std::vector<ScanSpan>> &spans, const ScanIndexRead &read, const MergeKeyRead &key,
                      const MergeSeek &seek, MergePlan *mp) {
    mp->cuts.clear();
    mp->refused = false;
    uint32_t live = 0;
    uint64_t n_spans = 0;
    for (uint32_t t = 0; t < n_tables; t++) {
        live += spans[t].empty() ? 0u : 1u;
        n_spans += spans[t].size();
    }
    const uint64_t step = std::max<uint64_t>(1, budget / (2ull * std::max(1u, live)));
    const bool span_starts = n_spans > kScanPartMaxSlices;
    struct Sample {
        uint32_t t, fs;
        uint64_t off;
    };
    std::vector<Sample> samples;
    std::vector<uint64_t> acc(n_tables, 0), max_fs(n_tables, 0);
    std::vector<size_t> next_span(n_tables, 0);
    const ScanRecordObserver obs = [&](uint32_t t, uint64_t r, uint64_t off, uint32_t fs) {
        const uint64_t b = (uint64_t)fs + 16;
        max_fs[t] = std::max<uint64_t>(max_fs[t], fs);
        bool take = acc[t] && acc[t] + b > step;
        while (next_span[t] < spans[t].size() && spans[t][next_span[t]].lo <= r) {
            take |= span_starts && spans[t][next_span[t]].lo == r && r > spans[t][0].lo;
            next_span[t]++;
        }
        if (take) {
            samples.push_back(Sample{t, fs, off});
            acc[t] = 0;
        }
        acc[t] += b;
    };
    int rc = plan_scan(data_len, index_len, n_tables, budget, read, &mp->plan, &spans, &obs);
    if (rc || mp->plan.panic_table >= 0 || mp->plan.parts.size() <= 1) return rc;
    uint64_t limit = budget; // the budget plus one record (and its index record) per table
    for (uint32_t t = 0; t < n_tables; t++) limit += spans[t].empty() ? 0 : max_fs[t] + 16;

    // ---- 2. splitters and the cuts of every table
    std::vector<std::vector<uint8_t>> keys;
    keys.reserve(samples.size());
    for (const Sample &x : samples) {
        std::vector<uint8_t> k;
        bool ok = false;
        if ((rc = key(x.t, x.off, x.fs, &k, &ok))) return rc;
        if (ok && !k.empty()) keys.push_back(std::move(k));
    }
    std::vector<Sample>().swap(samples);
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    std::vector<uint64_t> pos;
    if (!keys.empty() && (rc = seek(keys, &pos))) return rc;
    std::vector<std::vector<uint8_t>> split;
    std::vector<std::vector<uint64_t>> cut(n_tables);
    for (size_t j = 0; j < keys.size(); j++) {
        bool ok = true;
        for (uint32_t t = 0; t < n_tables; t++) ok &= spans[t].empty() || pos[(uint64_t)t * keys.size() + j] != ~0ull;
        if (!ok) continue;
        for (uint32_t t = 0; t < n_tables; t++) {
            const uint64_t n = index_len[t] / 16;
            uint64_t c = spans[t].empty() ? 0 : std::min(pos[(uint64_t)t * keys.size() + j], n);
            if (!cut[t].empty()) c = std::max(c, cut[t].back());
            cut[t].push_back(c);
        }
        split.push_back(std::move(keys[j]));
    }
    std::vector<std::vector<uint8_t>>().swap(keys);
    const uint32_t nk = (uint32_t)split.size();

    // ---- 3. pieces: the span records of one table, interval and span
    struct Piece {
        uint32_t iv, t;
        uint64_t rec_lo, rec_hi, win_lo, win_hi, bytes;
    };
    std::vector<Piece> pieces;
    std::vector<uint8_t> buf(kScanPlanPiece);
    for (uint32_t t = 0; t < n_tables; t++) {
        uint32_t iv = 0;
        bool open = false;
        Piece pc = {};
        for (const ScanSpan &span : spans[t]) {
            const uint64_t s_hi = std::min(span.hi, index_len[t] / 16);
            for (uint64_t r0 = span.lo; r0 < s_hi; r0 += kScanPlanPiece / 16) {
                const uint64_t m = std::min(s_hi - r0, kScanPlanPiece / 16);
                if ((rc = read(t, 16 * r0, 16 * m, buf.data()))) return rc;
                for (uint64_t k = 0; k < m; k++) {
                    const uint8_t *q = buf.data() + 16 * k;
                    const uint64_t r = r0 + k;
                    uint64_t off = 0;
                    uint32_t fs = 0;
                    for (int b = 7; b >= 0; b--) off = (off << 8) | q[b];
                    for (int b = 15; b >= 12; b--) fs = (fs << 8) | q[b];
                    while (iv < nk && cut[t][iv] <= r) iv++;
                    if (open && (pc.iv != iv || pc.rec_hi != r ||
                                 std::max(pc.win_hi, off + fs) - std::min(pc.win_lo, off) > pc.bytes + fs)) {
                        pieces.push_back(pc);
                        open = false;
                    }
                    if (!open) {
                        pc = Piece{iv, t, r, r, off, off + fs, 0};
                        open = true;
                    }
                    pc.rec_hi = r + 1;
                    pc.win_lo = std::min(pc.win_lo, off);
                    pc.win_hi = std::max(pc.win_hi, off + fs);
                    pc.bytes += fs;
                }
            }
        }
        if (open) pieces.push_back(pc);
    }
    std::stable_sort(pieces.begin(), pieces.end(), [](const Piece &a, const Piece &b) { return a.iv < b.iv; });

    // ---- 4. adjacent intervals merged up to the budget
    ScanPlan &plan = mp->plan;
    plan.parts.clear();
    plan.slices.clear();
    struct Open {
        ScanSlice sl;
        uint64_t bytes; // sum of full_size of its records: the bound on its window
    };
    std::map<uint32_t, std::vector<Open>> cur; // the open partition's slices per table
    uint64_t win = 0, out = 0, n_rec = 0, bound = 0;
    uint32_t n_sl = 0;
    auto emit = [&]() {
        ScanPart part{(uint32_t)plan.slices.size(), 0, n_rec, bound};
        for (const auto &kv : cur)
            for (const Open &o : kv.second) {
                plan.slices.push_back(o.sl);
                part.n_slices++;
            }
        plan.parts.push_back(part);
        cur.clear();
        win = out = n_rec = bound = 0;
        n_sl = 0;
    };
    auto joins = [&](const Piece &pc) -> Open * { // pc continues the table's last slice, within its bytes
        auto it = cur.find(pc.t);
        if (it == cur.end()) return nullptr;
        Open &b = it->second.back();
        const bool fits = std::max(b.sl.win_hi, pc.win_hi) - std::min(b.sl.win_lo, pc.win_lo) <= b.bytes + pc.bytes;
        return b.sl.rec_hi == pc.rec_lo && fits ? &b : nullptr;
    };
    for (size_t p = 0; p < pieces.size();) {
        const uint32_t iv = pieces[p].iv;
        size_t q = p;
        while (q < pieces.size() && pieces[q].iv == iv) q++;
        auto cost = [&](uint64_t *dw, uint64_t *dout, uint64_t *dn, uint32_t *ds) {
            *dw = *dout = *dn = 0;
            *ds = 0;
            for (size_t k = p; k < q; k++) {
                const Piece &pc = pieces[k];
                if (const Open *o = joins(pc)) {
                    const ScanSlice *b = &o->sl;
                    *dw += std::max(b->win_hi, pc.win_hi) - std::min(b->win_lo, pc.win_lo) - (b->win_hi - b->win_lo);
                }
                else {
                    *dw += pc.win_hi - pc.win_lo;
                    ++*ds;
                }
                *dout += pc.bytes + 16 * (pc.rec_hi - pc.rec_lo);
                *dn += pc.rec_hi - pc.rec_lo;
            }
        };
        uint64_t dw, dout, dn;
        uint32_t ds;
        cost(&dw, &dout, &dn, &ds);
        if (n_rec && (win + dw > budget || out + dout > budget || n_rec + dn > kScanPartMaxRecords || n_sl + ds > kScanPartMaxSlices)) {
            emit();
            mp->cuts.push_back(split[iv - 1]); // iv >= 1: an earlier interval holds records
            cost(&dw, &dout, &dn, &ds);
        }
        if (win + dw > limit || out + dout > limit || ds > kScanPartMaxSlices || dn > kScanPartMaxRecords) {
            plan.parts.clear();
            plan.slices.clear();
            mp->cuts.clear();
            mp->refused = true;
            return 0;
        }
        for (size_t k = p; k < q; k++) {
            const Piece &pc = pieces[k];
            if (Open *o = joins(pc)) {
                o->sl.rec_hi = pc.rec_hi;
                o->sl.win_lo = std::min(o->sl.win_lo, pc.win_lo);
                o->sl.win_hi = std::max(o->sl.win_hi, pc.win_hi);
                o->bytes += pc.bytes;
            } else {
                cur[pc.t].push_back(Open{ScanSlice{pc.t, pc.rec_lo, pc.rec_hi, pc.win_lo, pc.win_hi}, pc.bytes});
            }
            bound += pc.bytes;
        }
        win += dw;
        out += dout;
        n_rec += dn;
        n_sl += ds;
        p = q;
    }
    if (n_rec) emit();
    return 0;
}

} // namespace dbeel
