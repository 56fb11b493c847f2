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
#pragma once
#include <stdint.h>

#include <functional>
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

inline int plan_scan(const uint64_t *data_len, const uint64_t *index_len, uint32_t n_tables, uint64_t budget,
                     const ScanIndexRead &read, ScanPlan *plan) {
    plan->parts.clear();
    plan->slices.clear();
    plan->panic_table = -1;
    plan->panic_record = 0;
    std::vector<uint8_t> buf(kScanPlanPiece);
    bool open = false;        // a partition is being filled
    ScanPart part = {};
    ScanSlice sl = {};        // the open partition's last slice (its table is the current one once a record is in)
    bool slice_open = false;
    uint64_t closed_win = 0;  // windows of the open partition's earlier slices
    uint64_t out_bound = 0;   // sum of (full_size + 16) in the open partition
    auto close_slice = [&]() {
        if (!slice_open) return;
        plan->slices.push_back(sl);
        part.n_slices++;
        closed_win += sl.win_hi - sl.win_lo;
        slice_open = false;
    };
    auto close_part = [&]() {
        if (!open) return;
        close_slice();
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
        for (uint64_t r0 = 0; r0 < n; r0 += kScanPlanPiece / 16) {
            const uint64_t m = n - r0 < kScanPlanPiece / 16 ? n - r0 : kScanPlanPiece / 16;
            const int rc = read(t, 16 * r0, 16 * m, buf.data());
            if (rc) return rc;
            for (uint64_t k = 0; k < m; k++) {
                const uint8_t *q = buf.data() + 16 * k;
                uint64_t off = 0;
                uint32_t fs = 0;
                for (int b = 7; b >= 0; b--) off = (off << 8) | q[b];
                for (int b = 15; b >= 12; b--) fs = (fs << 8) | q[b];
                if (fs == 0 || off > data_len[t] || fs > data_len[t] - off) { // cached_file_reader.rs:68,82
                    plan->panic_table = (int32_t)t;
                    plan->panic_record = r0 + k;
                    close_part();
                    return 0;
                }
                const uint64_t lo = off, hi = off + fs;
                if (open) { // would this record push the partition past the budget?
                    const bool same = slice_open && sl.table == t;
                    const uint64_t w = same ? (hi > sl.win_hi ? hi : sl.win_hi) - (lo < sl.win_lo ? lo : sl.win_lo)
                                            : (slice_open ? sl.win_hi - sl.win_lo : 0) + fs;
                    if (closed_win + w > budget || out_bound + fs + 16 > budget || part.n_rec + 1 > kScanPartMaxRecords) close_part();
                }
                if (!open) {
                    part = ScanPart{(uint32_t)plan->slices.size(), 0, 0, 0};
                    closed_win = 0;
                    out_bound = 0;
                    open = true;
                }
                if (slice_open && sl.table != t) close_slice();
                if (!slice_open) {
                    sl = ScanSlice{t, r0 + k, r0 + k, lo, hi};
                    slice_open = true;
                }
                if (lo < sl.win_lo) sl.win_lo = lo;
                if (hi > sl.win_hi) sl.win_hi = hi;
                sl.rec_hi = r0 + k + 1;
                part.n_rec++;
                part.data_bound += fs;
                out_bound += fs + 16;
            }
        }
    }
    close_part();
    return 0;
}

} // namespace dbeel
