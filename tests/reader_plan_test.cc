// Host checks of the reader rules in dbeel_b200/csrc/host/lookup_plan.h (driven by tests/test_reader_plan_host.py):
//   depths    reader_depths over many table sets and budgets: never deeper than log2 n or kLookupMaxDepth, the fences of
//             all tables (both modes) fit fence_bytes, fixed depths are kept and counted, no table could take one more
//             level from what is left, 0 means the default budget, larger leaves get at least the depth of smaller ones
//   premise   the node states of a depth-D probe tree equal the top levels of every deeper one, both modes: a fence set
//             cached at D_t serves a batch at any depth <= D_t with the same comparisons in the same order
//   fallback  reader_uses_cache: the frame cap and the depth; lookup_depth grows with the number of open queries, so a
//             batch of n keys never wants more than lookup_depth(n, ...)
// Prints "ok" or the first mismatch.
#include <stdio.h>
#include <string.h>

#include <random>
#include <vector>

#include "../dbeel_b200/csrc/host/lookup_plan.h"

using namespace dbeel;

static uint64_t total(const std::vector<uint32_t> &d) {
    uint64_t s = 0;
    for (uint32_t x : d) s += reader_fence_bytes(x);
    return s;
}

static int check_set(const std::vector<uint64_t> &n, const std::vector<uint64_t> &len, const std::vector<int32_t> &fixed, uint64_t budget) {
    const std::vector<uint32_t> d = reader_depths(n, len, fixed, budget);
    const uint64_t b = budget ? budget : kReaderFenceBytesDefault;
    uint64_t fixed_bytes = 0;
    for (size_t t = 0; t < n.size(); t++)
        if (fixed[t] >= 0) fixed_bytes += reader_fence_bytes((uint32_t)fixed[t]);
    for (size_t t = 0; t < n.size(); t++) {
        if (fixed[t] >= 0 && d[t] != (uint32_t)fixed[t]) return printf("depths: table %zu lost its fixed depth\n", t), 1;
        if (d[t] > kLookupMaxDepth || d[t] > lookup_max_depth(n[t]) || (n[t] >= 1 && (1ull << d[t]) > n[t]))
            return printf("depths: table %zu of %llu records at depth %u\n", t, (unsigned long long)n[t], d[t]), 1;
    }
    if (fixed_bytes <= b && total(d) > b) return printf("depths: %llu bytes of fences over a budget of %llu\n", (unsigned long long)total(d), (unsigned long long)b), 1;
    const uint64_t left = b - std::min(b, total(d));
    for (size_t t = 0; t < n.size(); t++) {
        if (fixed[t] >= 0 || d[t] >= lookup_max_depth(n[t])) continue;
        if (reader_fence_bytes(d[t] + 1) - reader_fence_bytes(d[t]) <= left)
            return printf("depths: table %zu could go one level deeper (%u) within what is left\n", t, d[t]), 1;
        for (size_t u = 0; u < n.size(); u++) // the budget went to the larger leaves first
            if (fixed[u] < 0 && d[u] > d[t] + 1 && ((len[u] + 16 * n[u]) >> (d[u] - 1)) < ((len[t] + 16 * n[t]) >> d[t]))
                return printf("depths: table %zu deepened past table %zu whose leaves are larger\n", u, t), 1;
    }
    return 0;
}

static int depths() {
    // one table: the deepest level that fits, clamped by log2 n and 16
    for (uint64_t n : {0ull, 1ull, 2ull, 3ull, 100ull, 20000ull, 65536ull, 1ull << 20, 1ull << 30}) {
        for (uint64_t budget : {1ull, 415ull, 416ull, 4096ull, 1ull << 20, 64ull << 20, 1ull << 40}) {
            const std::vector<uint32_t> d = reader_depths({n}, {n * 100}, {-1}, budget);
            uint32_t want = 0;
            while (want < lookup_max_depth(n) && reader_fence_bytes(want + 1) <= budget) want++;
            if (d[0] != want) return printf("depths: n=%llu budget=%llu: %u, want %u\n", (unsigned long long)n, (unsigned long long)budget, d[0], want), 1;
        }
    }
    if (reader_depths({1ull << 30}, {1ull << 38}, {-1}, 0)[0] != lookup_max_depth(1ull << 30) ||
        reader_depths({1ull << 30}, {1ull << 38}, {-1}, 0) != reader_depths({1ull << 30}, {1ull << 38}, {-1}, kReaderFenceBytesDefault))
        return printf("depths: the default budget\n"), 1;
    if (reader_fence_bytes(16) != (2 * kReaderNodeBytes) << 16 || reader_fence_bytes(0) != 0) return printf("depths: fence bytes\n"), 1;
    // random table sets, some tables fixed by an earlier reader
    std::mt19937_64 rng(5);
    for (int it = 0; it < 3000; it++) {
        const size_t nt = 1 + rng() % 12;
        std::vector<uint64_t> n(nt), len(nt);
        std::vector<int32_t> fixed(nt, -1);
        for (size_t t = 0; t < nt; t++) {
            n[t] = rng() % 3 == 0 ? rng() % 50 : (1ull << (rng() % 34)) + rng() % 1000;
            len[t] = n[t] * (24 + rng() % 2000);
            if (rng() % 4 == 0) fixed[t] = (int32_t)std::min<uint32_t>(lookup_max_depth(n[t]), (uint32_t)(rng() % 10));
        }
        const uint64_t budget = rng() % 4 == 0 ? 0 : (rng() % 3 == 0 ? rng() % 100000 : rng() % (256ull << 20));
        if (check_set(n, len, fixed, budget)) return 1;
    }
    return 0;
}

static int premise() {
    for (uint32_t mode = 0; mode < 2; mode++)
        for (uint64_t n : {2ull, 3ull, 5ull, 17ull, 100ull, 1000ull, 20000ull, 65537ull, 1ull << 20, (1ull << 33) + 7}) {
            ProbeTree deep;
            plan_probe_tree(mode, n, lookup_max_depth(n), &deep);
            for (uint32_t d = 0; d < deep.depth; d++) {
                ProbeTree t;
                plan_probe_tree(mode, n, d, &t);
                for (uint64_t k = 1; k < (2ull << d); k++)
                    if (t.open[k] != deep.open[k] || (t.open[k] && memcmp(&t.state[k], &deep.state[k], sizeof(SearchState)) != 0))
                        return printf("premise: mode %u n=%llu depth %u node %llu\n", mode, (unsigned long long)n, d, (unsigned long long)k), 1;
            }
        }
    return 0;
}

static int fallback() {
    if (!reader_uses_cache(kReaderFrameCap, 5, 5) || !reader_uses_cache(0, 0, 0) || !reader_uses_cache(1, 3, 16))
        return printf("fallback: a batch the cache serves\n"), 1;
    if (reader_uses_cache(kReaderFrameCap + 1, 0, 16)) return printf("fallback: a key longer than the frame cap\n"), 1;
    if (reader_uses_cache(8, 6, 5)) return printf("fallback: a batch that wants more depth\n"), 1;
    if (kReaderFrameSlot < 8 + kReaderFrameCap || kReaderFrameSlot % 16) return printf("fallback: frame slot\n"), 1;
    // the decision made before the filter runs: lookup_depth(m) <= lookup_depth(n_keys) for every m <= n_keys
    for (uint64_t n : {2ull, 1000ull, 1ull << 20, 1ull << 32})
        for (uint64_t len : {n * 40, n * 5000})
            for (uint64_t budget : {4096ull, 1ull << 20, 256ull << 20}) {
                uint32_t prev = 0;
                for (uint64_t m = 0; m <= (1ull << 22); m = m ? m * 2 : 1) {
                    const uint32_t d = lookup_depth(m, n, len, 8 + 64, budget);
                    if (d < prev) return printf("fallback: lookup_depth shrinks with m at n=%llu m=%llu\n", (unsigned long long)n, (unsigned long long)m), 1;
                    prev = d;
                }
            }
    return 0;
}

int main(int argc, char **argv) {
    const char *what = argc > 1 ? argv[1] : "";
    if (!strcmp(what, "depths")) {
        if (depths()) return 1;
    } else if (!strcmp(what, "premise")) {
        if (premise()) return 1;
    } else if (!strcmp(what, "fallback")) {
        if (fallback()) return 1;
    } else {
        return printf("usage: depths | premise | fallback\n"), 2;
    }
    printf("ok\n");
    return 0;
}
