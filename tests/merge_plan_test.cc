// merge_plan_test.cc -- plan_merge (dbeel_b200/csrc/host/scan_plan.h), the key-aligned partition planner of
// dbeel_reader_get_range, on random in-memory tables with a host binary search as its seek:
//   * the partitions tile every table's spans exactly, in record order;
//   * every record of partition c has a key in [cuts[c - 1], cuts[c]) (tables whose keys ascend);
//   * every partition's windows and output bound are at most the budget plus one record per table;
//   * on tables with shuffled records the cuts stay monotone, so the partitions still tile the spans;
//   * on shuffled tables and on a sorted table with one index record pointed at another entry, the bound holds or the
//     planner refuses (MergePlan::refused) and plans nothing;
//   * spans that fit one partition cost no planner read: no key read, no seek, one pass over the span .index slices.
//
//   g++ -O2 -std=c++17 tests/merge_plan_test.cc -o /tmp/merge_plan_test && /tmp/merge_plan_test random|prefix|shuffled|one
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <random>
#include <string>

#include "../dbeel_b200/csrc/host/scan_plan.h"

using namespace dbeel;

namespace {

#define CHECK(c)                                                                 \
    do {                                                                         \
        if (!(c)) {                                                              \
            fprintf(stderr, "%s:%d: check failed: %s\n", __FILE__, __LINE__, #c); \
            exit(1);                                                             \
        }                                                                        \
    } while (0)

struct Table {
    std::vector<uint8_t> data, index;
    std::vector<std::vector<uint8_t>> keys; // per record (index order)
    std::vector<uint32_t> fs;
};

void put(std::vector<uint8_t> &v, uint64_t x, int n) {
    for (int b = 0; b < n; b++) v.push_back((uint8_t)(x >> (8 * b)));
}

Table make_table(std::vector<std::vector<uint8_t>> keys, std::mt19937_64 &rng, bool shuffle) {
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    Table t;
    std::vector<std::array<uint64_t, 2>> recs;
    for (const auto &k : keys) {
        const uint64_t dlen = rng() % 4 == 0 ? 0 : rng() % 200;
        const uint64_t off = t.data.size();
        put(t.data, k.size(), 8);
        t.data.insert(t.data.end(), k.begin(), k.end());
        put(t.data, dlen, 8);
        for (uint64_t j = 0; j < dlen + 16; j++) t.data.push_back((uint8_t)rng());
        recs.push_back({off, t.data.size() - off});
    }
    std::vector<size_t> order(keys.size());
    for (size_t j = 0; j < order.size(); j++) order[j] = j;
    if (shuffle) std::shuffle(order.begin(), order.end(), rng);
    for (size_t j : order) {
        put(t.index, recs[j][0], 8);
        put(t.index, 8 + keys[j].size(), 4);
        put(t.index, recs[j][1], 4);
        t.keys.push_back(keys[j]);
        t.fs.push_back((uint32_t)recs[j][1]);
    }
    return t;
}

std::vector<uint8_t> random_key(std::mt19937_64 &rng, const std::vector<uint8_t> &prefix, int len) {
    std::vector<uint8_t> k = prefix;
    while ((int)k.size() < len) k.push_back((uint8_t)(rng() % 4 == 0 ? 0 : rng() % 256));
    return k;
}

// seek_t of dbeel_reader_scan: a = 0, b = n; while a < b: mid, key(mid) < k ? a = mid + 1 : b = mid
uint64_t seek(const Table &t, const std::vector<uint8_t> &k) {
    uint64_t a = 0, b = t.keys.size();
    while (a < b) {
        const uint64_t mid = a + (b - a) / 2;
        if (t.keys[mid] < k) a = mid + 1; else b = mid;
    }
    return a;
}

struct Counts {
    uint64_t index_bytes = 0, key_reads = 0, seeks = 0;
};

MergePlan plan(const std::vector<Table> &ts, const std::vector<std::vector<ScanSpan>> &spans, uint64_t budget, Counts *cnt) {
    std::vector<uint64_t> dl, il;
    for (const Table &t : ts) {
        dl.push_back(t.data.size());
        il.push_back(t.index.size());
    }
    const ScanIndexRead rd = [&](uint32_t t, uint64_t off, uint64_t len, void *dst) {
        CHECK(off + len <= ts[t].index.size());
        memcpy(dst, ts[t].index.data() + off, len);
        cnt->index_bytes += len;
        return 0;
    };
    const MergeKeyRead key = [&](uint32_t t, uint64_t off, uint32_t fs, std::vector<uint8_t> *k, bool *ok) {
        CHECK(off + fs <= ts[t].data.size());
        uint64_t klen = 0;
        memcpy(&klen, ts[t].data.data() + off, 8);
        k->assign(ts[t].data.begin() + off + 8, ts[t].data.begin() + off + 8 + klen);
        *ok = true;
        cnt->key_reads++;
        return 0;
    };
    const MergeSeek sk = [&](const std::vector<std::vector<uint8_t>> &keys, std::vector<uint64_t> *pos) {
        CHECK(std::is_sorted(keys.begin(), keys.end()));
        pos->assign(ts.size() * keys.size(), 0);
        for (size_t t = 0; t < ts.size(); t++)
            for (size_t j = 0; j < keys.size(); j++) (*pos)[t * keys.size() + j] = seek(ts[t], keys[j]);
        cnt->seeks++;
        return 0;
    };
    MergePlan mp;
    CHECK(plan_merge(dl.data(), il.data(), (uint32_t)ts.size(), budget, spans, rd, key, sk, &mp) == 0);
    CHECK(!mp.refused || (mp.plan.parts.empty() && mp.plan.slices.empty() && mp.cuts.empty()));
    return mp;
}

// spans of random ranges: per table [seek(start), seek(end)) merged
std::vector<std::vector<ScanSpan>> random_spans(const std::vector<Table> &ts, std::mt19937_64 &rng, int n_ranges,
                                                const std::vector<uint8_t> &prefix, int klen) {
    std::vector<std::vector<ScanSpan>> spans(ts.size());
    std::vector<std::pair<std::vector<uint8_t>, std::vector<uint8_t>>> ranges;
    for (int d = 0; d < n_ranges; d++) {
        auto a = random_key(rng, prefix, klen), b = random_key(rng, prefix, klen);
        if (b < a) std::swap(a, b);
        ranges.push_back({a, b});
    }
    if (n_ranges == 0) ranges.push_back({{}, std::vector<uint8_t>(200, 0xFF)});
    for (size_t t = 0; t < ts.size(); t++) {
        std::vector<ScanSpan> sp;
        for (auto &r : ranges) {
            const uint64_t lo = seek(ts[t], r.first), hi = seek(ts[t], r.second);
            if (lo < hi) sp.push_back({lo, hi});
        }
        std::sort(sp.begin(), sp.end(), [](const ScanSpan &a, const ScanSpan &b) { return a.lo < b.lo; });
        for (const ScanSpan &x : sp) {
            if (!spans[t].empty() && x.lo <= spans[t].back().hi) spans[t].back().hi = std::max(spans[t].back().hi, x.hi);
            else spans[t].push_back(x);
        }
    }
    return spans;
}

void check_plan(const std::vector<Table> &ts, const std::vector<std::vector<ScanSpan>> &spans, uint64_t budget,
                const MergePlan &mp, bool sorted) {
    const ScanPlan &p = mp.plan;
    CHECK(p.panic_table < 0);
    CHECK(mp.cuts.size() + 1 == p.parts.size() || (p.parts.empty() && mp.cuts.empty()));
    CHECK(std::is_sorted(mp.cuts.begin(), mp.cuts.end()));
    std::vector<std::vector<uint64_t>> seen(ts.size());
    uint64_t max_fs_sum = 0;
    for (const Table &t : ts) max_fs_sum += t.fs.empty() ? 0 : *std::max_element(t.fs.begin(), t.fs.end());
    for (size_t c = 0; c < p.parts.size(); c++) {
        const ScanPart &pt = p.parts[c];
        CHECK(pt.n_slices > 0 && pt.n_slices <= kScanPartMaxSlices);
        uint64_t win = 0, out = 0, n = 0, bound = 0;
        int32_t last_t = -1;
        for (uint32_t k = 0; k < pt.n_slices; k++) {
            const ScanSlice &sl = p.slices[pt.first_slice + k];
            CHECK((int32_t)sl.table >= last_t);
            last_t = (int32_t)sl.table;
            CHECK(sl.rec_lo < sl.rec_hi);
            win += sl.win_hi - sl.win_lo;
            const Table &t = ts[sl.table];
            for (uint64_t r = sl.rec_lo; r < sl.rec_hi; r++) {
                uint64_t off = 0;
                memcpy(&off, t.index.data() + 16 * r, 8);
                CHECK(off >= sl.win_lo && off + t.fs[r] <= sl.win_hi);
                out += t.fs[r] + 16;
                bound += t.fs[r];
                n++;
                seen[sl.table].push_back(r);
                if (sorted) {
                    if (c > 0) CHECK(!(t.keys[r] < mp.cuts[c - 1]));
                    if (c + 1 < p.parts.size()) CHECK(t.keys[r] < mp.cuts[c]);
                }
            }
        }
        CHECK(n == pt.n_rec && bound == pt.data_bound);
        CHECK(win <= budget + max_fs_sum); // on any table: windows never pass their records' bytes
        CHECK(out <= budget + max_fs_sum + 16 * ts.size());
    }
    for (size_t t = 0; t < ts.size(); t++) { // the partitions tile the spans, in record order
        std::vector<uint64_t> want;
        for (const ScanSpan &x : spans[t])
            for (uint64_t r = x.lo; r < x.hi; r++) want.push_back(r);
        CHECK(seen[t] == want);
    }
}

int run(const char *mode) {
    std::mt19937_64 rng(12345);
    const bool prefix_mode = !strcmp(mode, "prefix"), shuffled = !strcmp(mode, "shuffled"), one = !strcmp(mode, "one");
    const bool damaged = !strcmp(mode, "damaged");
    int multi = 0, refused = 0;
    for (int it = 0; it < 60; it++) {
        const int n_tables = 1 + it % 6;
        const std::vector<uint8_t> prefix = prefix_mode ? std::vector<uint8_t>(80, 'P') : std::vector<uint8_t>{};
        const int klen = prefix_mode ? 100 : 1 + (int)(rng() % 12);
        std::vector<Table> ts;
        for (int t = 0; t < n_tables; t++) {
            std::vector<std::vector<uint8_t>> keys;
            const int n = 1 + (int)(rng() % (one ? 30 : 600));
            for (int j = 0; j < n; j++) keys.push_back(random_key(rng, prefix, prefix_mode ? klen : 1 + (int)(rng() % klen)));
            ts.push_back(make_table(keys, rng, shuffled && t == 1));
        }
        if (damaged) { // table 0: one index record's offset and full_size pointed at a far entry (a key out of order)
            Table &t = ts[0];
            const size_t n = t.keys.size(), a = n / 20, b = n - 1 - n / 20;
            if (n >= 2) {
                memcpy(t.index.data() + 16 * a, t.index.data() + 16 * b, 8);
                memcpy(t.index.data() + 16 * a + 8, t.index.data() + 16 * b + 8, 8);
                t.keys[a] = t.keys[b];
                t.fs[a] = t.fs[b];
            }
        }
        const int n_ranges = (int)(rng() % 4) == 0 ? 0 : 1 + (int)(rng() % (it % 3 == 0 ? 300 : 5));
        const auto spans = random_spans(ts, rng, n_ranges, prefix, prefix_mode ? klen : 3);
        for (uint64_t budget : {uint64_t(1) << 12, uint64_t(3000), uint64_t(1) << 15, uint64_t(1) << 30}) {
            if (one && budget < (1u << 30)) continue;
            Counts cnt;
            const MergePlan mp = plan(ts, spans, budget, &cnt);
            if (mp.refused) {
                CHECK(shuffled || damaged); // never on tables whose keys ascend
                refused++;
                continue;
            }
            check_plan(ts, spans, budget, mp, !shuffled && !damaged);
            uint64_t span_index = 0;
            for (const auto &s : spans)
                for (const ScanSpan &x : s) span_index += 16 * (x.hi - x.lo);
            ScanPlan flat; // plan_scan's plan of the same spans: one partition means no planner read
            std::vector<uint64_t> dl, il;
            for (const Table &t : ts) {
                dl.push_back(t.data.size());
                il.push_back(t.index.size());
            }
            CHECK(plan_scan(dl.data(), il.data(), (uint32_t)ts.size(), budget,
                            [&](uint32_t t, uint64_t off, uint64_t len, void *dst) {
                                memcpy(dst, ts[t].index.data() + off, len);
                                return 0;
                            }, &flat, &spans) == 0);
            if (flat.parts.size() <= 1) {
                CHECK(mp.plan.parts.size() == flat.parts.size() && mp.cuts.empty());
                CHECK(cnt.key_reads == 0 && cnt.seeks == 0 && cnt.index_bytes == span_index);
            } else {
                multi += mp.plan.parts.size() > 1;
                CHECK(cnt.index_bytes == 2 * span_index);
            }
        }
    }
    if (!one) CHECK(multi > 20);
    if (shuffled) CHECK(refused > 0); // a damaged offset only starts a new slice: the bound holds
    printf("multi %d refused %d\nok\n", multi, refused);
    return 0;
}

} // namespace

int main(int argc, char **argv) {
    if (argc == 2) return run(argv[1]);
    fprintf(stderr, "usage: %s random | prefix | shuffled | damaged | one\n", argv[0]);
    return 2;
}
