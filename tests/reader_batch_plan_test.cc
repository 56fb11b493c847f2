// Host checks of the leaf grouping of dbeel_readers_get_values (group_leaves over pairs, dbeel_b200/csrc/host/lookup_plan.h),
// driven by tests/test_reader_batch_plan_host.py, on random levels of (batch, table) pairs with and without page caches:
//   cover   the cuts start at 0, end at the last leaf and ascend: every touched leaf lands in exactly one group
//   solo    every cut inside a pair's leaves that its solo call makes (group_leaves on its leaves alone, with min(budget,
//           its cache) when paged) is a cut of the level, so a pair's reads are a subset of its solo call's
//   budget  a group of more than one solo unit keeps its estimate within the budget, and the leaves of each cache within
//           its capacity when they are more than one unit (one larger unit goes uncached, as in its solo call)
//   single  one pair gives exactly group_leaves' cuts
// Prints "ok" or the first mismatch.
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <random>
#include <vector>

#include "../dbeel_b200/csrc/host/lookup_plan.h"

using namespace dbeel;

struct Level {
    std::vector<TouchedLeaf> lv;
    std::vector<LeafPair> pairs;
    std::vector<uint64_t> cache_bytes;
    uint64_t budget;
};

static Level random_level(std::mt19937_64 &rng, uint32_t max_pairs) {
    Level L;
    const uint32_t np = 1 + rng() % max_pairs, nc = rng() % 4;
    for (uint32_t c = 0; c < nc; c++) L.cache_bytes.push_back(kPageBytes * (1 + rng() % 64));
    L.budget = 4096ull << (rng() % 10);
    for (uint32_t p = 0; p < np; p++) {
        const uint64_t n = rng() % 3 ? rng() % 100000 : rng() % 8;
        const uint64_t dl = n * (24 + rng() % 400);
        const int32_t cache = nc && rng() % 3 ? (int32_t)(rng() % nc) : -1;
        L.pairs.push_back(LeafPair{n, dl, 1 + rng() % 80, cache});
        if (rng() % 5 == 0 || n == 0) continue; // a pair no query reached
        const uint32_t depth = lookup_max_depth(n) ? rng() % (lookup_max_depth(n) + 1) : 0;
        const uint64_t leaves = 1ull << depth;
        for (uint64_t l = 0; l < leaves; l++) {
            if (rng() % 3) continue;
            const uint64_t a = n * l / leaves, b = n * (l + 1) / leaves;
            L.lv.push_back(TouchedLeaf{p, (uint32_t)l, a, std::max(b, a + 1)});
        }
    }
    return L;
}

// the solo call's cuts of pair p, as leaf indices of the level
static std::vector<size_t> solo_cuts(const Level &L, uint32_t p, size_t *k0_out) {
    size_t k0 = 0, k1;
    while (k0 < L.lv.size() && L.lv[k0].t != p) k0++;
    for (k1 = k0; k1 < L.lv.size() && L.lv[k1].t == p; k1++) {}
    std::vector<TouchedLeaf> mine(L.lv.begin() + k0, L.lv.begin() + k1);
    for (TouchedLeaf &l : mine) l.t = 0;
    const LeafPair &lp = L.pairs[p];
    const bool paged = lp.cache >= 0;
    std::vector<size_t> c = group_leaves(mine, {lp.n}, {lp.data_len}, lp.max_klen, paged ? std::min(L.budget, L.cache_bytes[lp.cache]) : L.budget, paged);
    for (size_t &x : c) x += k0;
    *k0_out = k0;
    return c;
}

static int check(const Level &L, const char *what) {
    const std::vector<size_t> cut = group_leaves(L.lv, L.pairs, L.budget, L.cache_bytes);
    if (!strcmp(what, "cover")) {
        if (L.lv.empty()) return cut != std::vector<size_t>{0} ? (printf("cover: cuts of no leaves\n"), 1) : 0;
        if (cut.front() != 0 || cut.back() != L.lv.size()) return printf("cover: cuts do not span the leaves\n"), 1;
        for (size_t g = 0; g + 1 < cut.size(); g++)
            if (cut[g] >= cut[g + 1]) return printf("cover: empty or descending group %zu\n", g), 1;
        return 0;
    }
    std::vector<uint8_t> is_unit(L.lv.size() + 1, 0); // a solo cut of some pair
    for (uint32_t p = 0; p < L.pairs.size(); p++) {
        size_t k0;
        const std::vector<size_t> sc = solo_cuts(L, p, &k0);
        for (size_t x : sc) {
            is_unit[x] = 1;
            if (x == sc.front() || x == sc.back()) continue; // where the pair's leaves start and end: shared with other pairs
            if (!strcmp(what, "solo") && !std::binary_search(cut.begin(), cut.end(), x))
                return printf("solo: pair %u's solo cut at leaf %zu is not a cut of the level\n", p, x), 1;
        }
    }
    if (!strcmp(what, "budget")) {
        for (size_t g = 0; g + 1 < cut.size(); g++) {
            uint64_t est = 0, units = 0;
            std::vector<uint64_t> est_c(L.cache_bytes.size(), 0), units_c(L.cache_bytes.size(), 0);
            for (size_t k = cut[g]; k < cut[g + 1]; k++) {
                const TouchedLeaf &l = L.lv[k];
                const LeafPair &lp = L.pairs[l.t];
                const uint64_t b = leaf_bytes(l, lp.n, lp.data_len, lp.max_klen, lp.cache >= 0);
                est += b;
                units += is_unit[k];
                if (lp.cache < 0) continue;
                est_c[lp.cache] += b;
                units_c[lp.cache] += is_unit[k];
            }
            if (units <= 1) continue;
            if (est > L.budget) return printf("budget: group %zu of %llu units holds %llu bytes over %llu\n", g, (unsigned long long)units, (unsigned long long)est, (unsigned long long)L.budget), 1;
            for (size_t c = 0; c < est_c.size(); c++) // one unit larger than its cache alone is read uncached, as solo
                if (units_c[c] > 1 && est_c[c] > L.cache_bytes[c]) return printf("budget: group %zu holds %llu bytes of cache %zu\n", g, (unsigned long long)est_c[c], c), 1;
        }
    }
    return 0;
}

static int single(std::mt19937_64 &rng) {
    for (int it = 0; it < 3000; it++) {
        Level L = random_level(rng, 1);
        const std::vector<size_t> cut = group_leaves(L.lv, L.pairs, L.budget, L.cache_bytes);
        const LeafPair &lp = L.pairs[0];
        const bool paged = lp.cache >= 0;
        const uint64_t gb = paged ? std::min(L.budget, L.cache_bytes[lp.cache]) : L.budget;
        if (cut != group_leaves(L.lv, {lp.n}, {lp.data_len}, lp.max_klen, gb, paged))
            return printf("single: one pair's cuts differ from group_leaves' (iteration %d)\n", it), 1;
    }
    return 0;
}

int main(int argc, char **argv) {
    const char *what = argc > 1 ? argv[1] : "";
    std::mt19937_64 rng(0x5EED);
    if (!strcmp(what, "single")) {
        if (single(rng)) return 1;
    } else if (!strcmp(what, "cover") || !strcmp(what, "solo") || !strcmp(what, "budget")) {
        for (int it = 0; it < 3000; it++)
            if (check(random_level(rng, 1 + it % 40), what)) return printf("(iteration %d)\n", it), 1;
    } else {
        return printf("usage: cover | solo | budget | single\n"), 2;
    }
    printf("ok\n");
    return 0;
}
