// Host checks of dbeel_b200/csrc/host/lookup_plan.h (driven by tests/test_lookup_plan_host.py):
//   descent  for every n in 0..600 and sampled large n (index offsets past 2^32), both modes, every depth: the fence descent
//            over the planned probe tree, then the resume from the leaf state, probes exactly the records the whole-table
//            loop of lookup.cuh probes and ends the same way, for present keys, absent keys between and around them, and the
//            reference's early exit; the rest of the search stays inside the leaf's interval
//   oracle   the whole-table loop of reference mode against the oracle's orc_sstable_lookup (oracle/dbeel_oracle.c,
//            linked in) on real tables of n = 0..300 records, for every present key and every gap
//   windows  leaf windows on damaged index slices: lying key_size / offset / full_size, overlapping records, full_size < 8
//   merge    merging of read ranges
// Prints "ok" or the first mismatch.  Table key of record r: 2r + 2, queries are integers (absent: odd or out of range).
#include <stdio.h>
#include <string.h>

#include <random>
#include <vector>

#include "../dbeel_b200/csrc/host/lookup_plan.h"

using namespace dbeel;

extern "C" {
typedef struct orc_run {
    const uint8_t *data;
    uint64_t data_len;
    const uint8_t *index;
    uint64_t index_len;
} orc_run;
int orc_sstable_lookup(const orc_run *run, const uint8_t *bloom, uint64_t bloom_len, const uint8_t *key, uint64_t klen,
                       uint64_t *record, int *bloom_said_no);
}

static int cmp_rec(uint64_t r, uint64_t q) { // the table key of record r against the query
    const uint64_t k = 2 * r + 2;
    return k < q ? -1 : (k > q ? 1 : 0);
}

// lookup_query's loops restated (lookup.cuh): returns the record found or -1, the probes in *seq
static int64_t whole(uint32_t mode, uint64_t n, uint64_t q, std::vector<uint64_t> *seq) {
    seq->clear();
    if (n == 0) return -1;
    if (mode == 0) {
        uint64_t half = n / 2, high = n - 1, low = 0;
        bool done = false;
        int64_t found = -1;
        while (!done) {
            seq->push_back(half);
            const int c = cmp_rec(half, q);
            if (c == 0) found = (int64_t)half;
            low = c < 0 ? half + 1 : low;
            high = c > 0 ? (half > 1 ? half : 1) - 1 : high;
            done = c == 0 || half == 0 || half == n;
            half = (high + low) / 2;
            done = done || low > high;
        }
        return found;
    }
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        seq->push_back(mid);
        const int c = cmp_rec(mid, q);
        if (c == 0) return (int64_t)mid;
        if (c < 0) lo = mid + 1; else hi = mid;
    }
    return -1;
}

// fence descent on the planned tree, then the resume from the leaf's state
static int64_t split(const ProbeTree &t, uint64_t q, std::vector<uint64_t> *seq, bool *ok) {
    seq->clear();
    *ok = true;
    SearchState s = search_init(t.mode, t.n);
    if (s.done) return -1;
    uint64_t node = 1;
    const uint64_t leaf0 = 1ull << t.depth;
    while (node < leaf0) {
        if (!t.open[node] || search_pos(t.mode, t.state[node]) != search_pos(t.mode, s)) { *ok = false; return -2; }
        const uint64_t p = search_pos(t.mode, s);
        seq->push_back(p);
        const int c = cmp_rec(p, q);
        if (c == 0) return (int64_t)p;
        search_step(t.mode, t.n, &s, c);
        if (s.done) return -1;
        node = 2 * node + (c < 0 ? 1 : 0);
    }
    if (!t.open[node] || memcmp(&t.state[node], &s, sizeof s) != 0) { *ok = false; return -2; }
    uint64_t lo, hi;
    search_interval(t.mode, s, &lo, &hi);
    while (!s.done) {
        const uint64_t p = search_pos(t.mode, s);
        if (p < lo || p >= hi) { *ok = false; return -2; }
        seq->push_back(p);
        const int c = cmp_rec(p, q);
        if (c == 0) return (int64_t)p;
        search_step(t.mode, t.n, &s, c);
    }
    return -1;
}

static int check_n(uint64_t n, const std::vector<uint64_t> &queries) {
    uint32_t dmax = 0;
    while (dmax < kLookupMaxDepth && (2ull << dmax) <= n) dmax++;
    std::vector<uint64_t> a, b;
    for (uint32_t mode = 0; mode < 2; mode++)
        for (uint32_t d = 0; d <= dmax; d++) {
            ProbeTree t;
            plan_probe_tree(mode, n, d, &t);
            for (uint64_t q : queries) {
                bool ok;
                const int64_t w = whole(mode, n, q, &a), s = split(t, q, &b, &ok);
                if (!ok || w != s || a != b) {
                    printf("MISMATCH n=%llu mode=%u depth=%u q=%llu whole=%lld split=%lld probes %zu/%zu\n", (unsigned long long)n,
                           mode, d, (unsigned long long)q, (long long)w, (long long)s, a.size(), b.size());
                    return 1;
                }
            }
        }
    return 0;
}

// Record r of a real table holds the 8-byte big-endian key 2r + 2 (so byte order is number order), an empty value and
// timestamp 0: u64 8 | key | u64 0 | i128 0 = 40 bytes.
static int oracle() {
    std::vector<uint64_t> seq;
    for (uint64_t n = 0; n <= 300; n++) {
        std::vector<uint8_t> data(40 * n + 8, 0), index(16 * n + 16, 0);
        for (uint64_t r = 0; r < n; r++) {
            uint8_t *e = data.data() + 40 * r;
            e[0] = 8;
            for (int b = 0; b < 8; b++) e[8 + b] = (uint8_t)((2 * r + 2) >> (56 - 8 * b));
            const uint64_t off = 40 * r;
            const uint32_t ks = 16, fs = 40;
            memcpy(index.data() + 16 * r, &off, 8);
            memcpy(index.data() + 16 * r + 8, &ks, 4);
            memcpy(index.data() + 16 * r + 12, &fs, 4);
        }
        const orc_run run = {data.data(), 40 * n, index.data(), 16 * n};
        for (uint64_t q = 0; q <= 2 * n + 3; q++) {
            uint8_t key[8];
            for (int b = 0; b < 8; b++) key[b] = (uint8_t)(q >> (56 - 8 * b));
            uint64_t rec = 0;
            int no = 0;
            const int found = orc_sstable_lookup(&run, nullptr, 0, key, 8, &rec, &no);
            const int64_t w = whole(0, n, q, &seq);
            if ((found != 0) != (w >= 0) || (found && (int64_t)rec != w)) {
                printf("ORACLE n=%llu q=%llu: oracle %d/%llu, loop %lld\n", (unsigned long long)n, (unsigned long long)q, found,
                       (unsigned long long)rec, (long long)w);
                return 1;
            }
        }
    }
    return 0;
}

static void put_rec(uint8_t *p, uint64_t off, uint32_t ks, uint32_t fs) {
    memcpy(p, &off, 8);
    memcpy(p + 8, &ks, 4);
    memcpy(p + 12, &fs, 4);
}

static int windows() {
    uint8_t s[16 * 4];
    ByteRange w;
    put_rec(s, 100, 20, 50); put_rec(s + 16, 150, 20, 50); put_rec(s + 32, 200, 20, 50);
    // running offsets: from the first record to the end of the last entry (each could answer a 12-byte query)
    if (!leaf_window(s, 3, 1000, 12, &w) || w.lo != 100 || w.hi != 250) return printf("window: running %llu %llu\n", (unsigned long long)w.lo, (unsigned long long)w.hi), 1;
    // key_size lies: no query can hit the record, so only its probe frame counts, not full_size
    put_rec(s + 32, 200, 900, 50);
    if (!leaf_window(s, 3, 1000, 12, &w) || w.hi != 220) return printf("window: key_size %llu\n", (unsigned long long)w.hi), 1;
    // full_size lies but stays inside .data: the whole claimed entry is in the window (a hit copies it); past .data: frame only
    put_rec(s + 32, 200, 20, 700);
    if (!leaf_window(s, 3, 1000, 12, &w) || w.hi != 900) return printf("window: full_size %llu\n", (unsigned long long)w.hi), 1;
    put_rec(s + 32, 200, 20, 900);
    if (!leaf_window(s, 3, 1000, 12, &w) || w.hi != 220) return printf("window: full_size past .data %llu\n", (unsigned long long)w.hi), 1;
    // an offset that lies backwards and one past the file: the window covers the first, skips the second
    put_rec(s, 100, 20, 50); put_rec(s + 16, 10, 20, 50); put_rec(s + 32, 995, 20, 50);
    if (!leaf_window(s, 3, 1000, 12, &w) || w.lo != 10 || w.hi != 150) return printf("window: offsets %llu %llu\n", (unsigned long long)w.lo, (unsigned long long)w.hi), 1;
    // a frame cut at the end of .data; overlapping records; full_size < 8 is not looked at
    put_rec(s, 990, 20, 3); put_rec(s + 16, 985, 20, 4); put_rec(s + 32, 988, 20, 2);
    if (!leaf_window(s, 3, 1000, 12, &w) || w.lo != 985 || w.hi != 1000) return printf("window: end\n"), 1;
    // every record past the file: no window
    put_rec(s, 1000, 20, 3); put_rec(s + 16, 993, 20, 4); put_rec(s + 32, ~0ull, 20, 2);
    if (leaf_window(s, 3, 1000, 12, &w)) return printf("window: none\n"), 1;
    // offsets past 2^32
    put_rec(s, (1ull << 32) + 5, 20, 50);
    if (!leaf_window(s, 1, 1ull << 33, 4, &w) || w.lo != (1ull << 32) + 5 || w.hi != (1ull << 32) + 17) return printf("window: far\n"), 1;
    return 0;
}

static int merge() {
    std::vector<ByteRange> r = {{50, 60}, {0, 10}, {12, 20}, {20, 30}, {5, 8}, {100, 200}, {150, 160}, {1ull << 33, (1ull << 33) + 1}};
    std::vector<ByteRange> m = merge_ranges(r, 0);
    const std::vector<ByteRange> want0 = {{0, 10}, {12, 30}, {50, 60}, {100, 200}, {1ull << 33, (1ull << 33) + 1}};
    if (m.size() != want0.size()) return printf("merge: gap 0 gives %zu\n", m.size()), 1;
    for (size_t k = 0; k < m.size(); k++)
        if (m[k].lo != want0[k].lo || m[k].hi != want0[k].hi) return printf("merge: gap 0 range %zu\n", k), 1;
    m = merge_ranges(r, 20);
    if (m.size() != 3 || m[0].lo != 0 || m[0].hi != 60 || m[1].lo != 100 || m[1].hi != 200) return printf("merge: gap 20\n"), 1;
    if (!merge_ranges({}, 5).empty()) return printf("merge: empty\n"), 1;
    return 0;
}

int main(int argc, char **argv) {
    const char *what = argc > 1 ? argv[1] : "";
    if (!strcmp(what, "descent")) {
        for (uint64_t n = 0; n <= 600; n++) {
            std::vector<uint64_t> qs;
            for (uint64_t q = 0; q <= 2 * n + 3; q++) qs.push_back(q); // every present key, every gap, both ends
            if (check_n(n, qs)) return 1;
        }
        std::mt19937_64 rng(7);
        for (uint64_t n : {1000ull, 65535ull, 65536ull, 65537ull, 1ull << 20, (1ull << 28) + 3, 300000007ull, (1ull << 36) + 1}) {
            std::vector<uint64_t> qs = {0, 1, 2, 3, 4, 2 * n, 2 * n + 1, 2 * n + 2, 2 * n + 3};
            for (int k = 0; k < 40; k++) qs.push_back(rng() % (2 * n + 4));
            if (check_n(n, qs)) return 1;
        }
    } else if (!strcmp(what, "oracle")) {
        if (oracle()) return 1;
    } else if (!strcmp(what, "windows")) {
        if (windows()) return 1;
    } else if (!strcmp(what, "merge")) {
        if (merge()) return 1;
    } else if (!strcmp(what, "depth")) {
        // the depth stays inside its clamps
        for (uint64_t n : {0ull, 1ull, 2ull, 3ull, 1000ull, 1ull << 30})
            for (uint64_t m : {0ull, 1ull, 1000ull, 1ull << 22}) {
                const uint32_t d = lookup_depth(m, n, n * 300, 24, 256ull << 20);
                if (d > kLookupMaxDepth || (n >= 1 && (1ull << d) > n) || ((m == 0 || n < 2) && d != 0)) return printf("depth n=%llu m=%llu: %u\n", (unsigned long long)n, (unsigned long long)m, d), 1;
            }
        if (lookup_depth(1000, 1ull << 30, 300ull << 30, 24, 256ull << 20) != 16) return printf("depth: large table\n"), 1;
        if (lookup_depth(1, 1ull << 20, 1ull << 28, 24, 1ull << 30) >= lookup_depth(1ull << 20, 1ull << 20, 1ull << 28, 24, 1ull << 30))
            return printf("depth: does not grow with the batch\n"), 1;
    } else {
        return printf("usage: descent | oracle | windows | merge | depth\n"), 2;
    }
    printf("ok\n");
    return 0;
}
