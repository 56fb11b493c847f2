// Host checks of the packing of dbeel_readers_get_ranges (pack_batches, dbeel_b200/csrc/host/lookup_plan.h): how the seek
// batches and the merge-round query groups of many batches share one search or one round.  Driven by
// tests/test_range_batch_plan_host.py, on random batches of unit costs with and without page caches:
//   cover   the groups hold every unit of every batch exactly once, in batch order, then unit order
//   solo    every group's span of a batch is one of that batch's solo groups (pack_in_order with the budget alone)
//   budget  a group of more than one span keeps its bytes within the budget, and each cache's bytes within its capacity
//   single  one batch gives exactly its solo groups
// Prints "ok" or the first mismatch.
#include <stdio.h>
#include <string.h>

#include <random>
#include <vector>

#include "../dbeel_b200/csrc/host/lookup_plan.h"

using namespace dbeel;

struct Case {
    std::vector<std::vector<uint64_t>> cost;
    std::vector<int32_t> cache;
    std::vector<uint64_t> cache_bytes;
    uint64_t budget;
};

static Case random_case(std::mt19937_64 &rng, uint32_t max_batches) {
    Case c;
    const uint32_t nb = 1 + rng() % max_batches, nc = rng() % 3;
    c.budget = 256 + rng() % 8192;
    for (uint32_t k = 0; k < nc; k++) c.cache_bytes.push_back(128 + rng() % 16384);
    for (uint32_t b = 0; b < nb; b++) {
        c.cost.emplace_back();
        const uint32_t n = rng() % 4 == 0 ? 0 : rng() % 40;
        for (uint32_t k = 0; k < n; k++) c.cost.back().push_back(rng() % 3 == 0 ? rng() % (2 * c.budget) : 1 + rng() % 400);
        c.cache.push_back(nc && rng() % 2 ? (int32_t)(rng() % nc) : -1);
    }
    return c;
}

static uint64_t span_bytes(const Case &c, const BatchSpan &s) {
    uint64_t x = 0;
    for (size_t k = s.k0; k < s.k1; k++) x += c.cost[s.batch][k];
    return x;
}

static bool check(const Case &c, const char *what) {
    const std::vector<std::vector<BatchSpan>> g = pack_batches(c.cost, c.cache, c.budget, c.cache_bytes);
    if (!strcmp(what, "cover")) {
        uint32_t b = 0;
        size_t k = 0;
        for (const auto &grp : g) {
            if (grp.empty()) return false;
            for (const BatchSpan &s : grp) {
                while (b < s.batch) {
                    if (k != c.cost[b].size()) return false;
                    b++, k = 0;
                }
                if (s.batch != b || s.k0 != k || s.k1 <= s.k0) return false;
                k = s.k1;
            }
        }
        for (; b < c.cost.size(); b++, k = 0)
            if (k != c.cost[b].size()) return false;
        return true;
    }
    if (!strcmp(what, "solo")) {
        for (const auto &grp : g)
            for (const BatchSpan &s : grp) {
                const std::vector<size_t> cut = pack_in_order(c.cost[s.batch], c.budget);
                bool found = false;
                for (size_t j = 0; j + 1 < cut.size(); j++) found |= cut[j] == s.k0 && cut[j + 1] == s.k1;
                if (!found) return false;
            }
        return true;
    }
    if (!strcmp(what, "budget")) {
        for (const auto &grp : g) {
            if (grp.size() < 2) continue;
            uint64_t est = 0;
            std::vector<uint64_t> est_c(c.cache_bytes.size(), 0);
            for (const BatchSpan &s : grp) {
                est += span_bytes(c, s);
                if (c.cache[s.batch] >= 0) est_c[c.cache[s.batch]] += span_bytes(c, s);
            }
            if (est > c.budget) return false;
            for (size_t k = 0; k < est_c.size(); k++) {
                uint32_t spans = 0;
                for (const BatchSpan &s : grp) spans += c.cache[s.batch] == (int32_t)k;
                if (spans > 1 && est_c[k] > c.cache_bytes[k]) return false;
            }
        }
        return true;
    }
    if (!strcmp(what, "single")) {
        if (c.cost.size() != 1) return true;
        const std::vector<size_t> cut = pack_in_order(c.cost[0], c.budget);
        if (g.size() + 1 != cut.size() && !(g.empty() && cut.size() == 1)) return false;
        for (size_t j = 0; j < g.size(); j++)
            if (g[j].size() != 1 || g[j][0].k0 != cut[j] || g[j][0].k1 != cut[j + 1]) return false;
        return true;
    }
    return false;
}

int main(int argc, char **argv) {
    if (argc != 2) return 2;
    std::mt19937_64 rng(20261018);
    for (int it = 0; it < 20000; it++) {
        const Case c = random_case(rng, strcmp(argv[1], "single") ? 12 : 1);
        if (!check(c, argv[1])) {
            printf("%s: mismatch at case %d (%zu batches, budget %llu)\n", argv[1], it, c.cost.size(), (unsigned long long)c.budget);
            return 1;
        }
    }
    printf("%s ok\n", argv[1]);
    return 0;
}
