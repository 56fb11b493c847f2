// scan_seek_host_test.cc -- plan_scan with record spans (dbeel_reader_scan's key ranges, dbeel_b200/csrc/host/scan_plan.h)
// on a box without a GPU; driven by tests/test_scan_seek_host.py.
//
//   spans B1 B2 ...   reads a tree from stdin ("n_tables", then per table "data_len index_path n_spans lo hi lo hi ..."),
//                     and at every budget checks
//                       * plan_scan with spans == plan_scan over the tables cut down to their spans (each .index = its
//                         span records back to back; a table with records but no span dropped), record numbers mapped
//                         back: the same partitions and PANIC, every cut slice split at span boundaries, each piece with
//                         the window of its own records;
//                       * plan_scan with one whole-table span per table == plan_scan with no spans;
//                       * the span plan reads only span slices, in pieces of at most 1 MiB.
//                     Prints "ok" or the first difference.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../dbeel_b200/csrc/host/scan_plan.h"

namespace {

using dbeel::ScanPlan;
using dbeel::ScanSlice;
using dbeel::ScanSpan;

struct Tree {
    std::vector<uint64_t> dlen, ilen;
    std::vector<std::vector<uint8_t>> index;
    std::vector<std::vector<ScanSpan>> spans;
};

uint64_t rd(const uint8_t *p, int nb) {
    uint64_t v = 0;
    for (int b = nb - 1; b >= 0; b--) v = (v << 8) | p[b];
    return v;
}

bool same_plan(const ScanPlan &a, const ScanPlan &b, const char *what, uint64_t budget) {
    bool ok = a.panic_table == b.panic_table && a.panic_record == b.panic_record && a.parts.size() == b.parts.size() &&
              a.slices.size() == b.slices.size();
    for (size_t k = 0; ok && k < a.parts.size(); k++)
        ok = a.parts[k].first_slice == b.parts[k].first_slice && a.parts[k].n_slices == b.parts[k].n_slices &&
             a.parts[k].n_rec == b.parts[k].n_rec && a.parts[k].data_bound == b.parts[k].data_bound;
    for (size_t k = 0; ok && k < a.slices.size(); k++)
        ok = a.slices[k].table == b.slices[k].table && a.slices[k].rec_lo == b.slices[k].rec_lo && a.slices[k].rec_hi == b.slices[k].rec_hi &&
             a.slices[k].win_lo == b.slices[k].win_lo && a.slices[k].win_hi == b.slices[k].win_hi;
    if (!ok) {
        printf("%s differ at budget %llu: parts %zu / %zu, slices %zu / %zu, panic %d %llu / %d %llu\n", what, (unsigned long long)budget,
               a.parts.size(), b.parts.size(), a.slices.size(), b.slices.size(), a.panic_table, (unsigned long long)a.panic_record,
               b.panic_table, (unsigned long long)b.panic_record);
    }
    return ok;
}

int run_spans(int argc, char **argv) {
    uint32_t n = 0;
    if (scanf("%u", &n) != 1) return 2;
    Tree tr;
    tr.dlen.resize(n);
    tr.ilen.resize(n);
    tr.index.resize(n);
    tr.spans.resize(n);
    for (uint32_t t = 0; t < n; t++) {
        unsigned long long dl;
        char path[4096];
        unsigned ns;
        if (scanf("%llu %4095s %u", &dl, path, &ns) != 3) return 2;
        for (unsigned k = 0; k < ns; k++) {
            unsigned long long lo, hi;
            if (scanf("%llu %llu", &lo, &hi) != 2) return 2;
            tr.spans[t].push_back(ScanSpan{lo, hi});
        }
        tr.dlen[t] = dl;
        FILE *fp = fopen(path, "rb");
        if (!fp) return 3;
        uint8_t b[65536];
        size_t r;
        while ((r = fread(b, 1, sizeof b, fp)) > 0) tr.index[t].insert(tr.index[t].end(), b, b + r);
        fclose(fp);
        tr.ilen[t] = tr.index[t].size();
    }
    // the cut tree: cut table c = original table orig[c]; cut record i = original record map[c][i]
    std::vector<uint32_t> orig;
    std::vector<std::vector<uint64_t>> map;
    std::vector<std::vector<uint8_t>> cut_index;
    std::vector<uint64_t> cdlen, cilen;
    for (uint32_t t = 0; t < n; t++) {
        const uint64_t nrec = tr.ilen[t] / 16;
        std::vector<uint64_t> m;
        std::vector<uint8_t> ix;
        for (const ScanSpan &s : tr.spans[t])
            for (uint64_t r = s.lo; r < std::min(s.hi, nrec); r++) {
                m.push_back(r);
                ix.insert(ix.end(), tr.index[t].begin() + 16 * r, tr.index[t].begin() + 16 * r + 16);
            }
        if (nrec && m.empty()) continue; // a table with records but an empty span contributes nothing
        orig.push_back(t);
        map.push_back(m);
        cut_index.push_back(ix);
        cdlen.push_back(tr.dlen[t]);
        cilen.push_back(ix.size());
    }
    uint64_t max_read = 0;
    bool outside = false;
    auto read = [&](uint32_t t, uint64_t off, uint64_t len, void *dst) {
        if (off + len > tr.index[t].size()) return 5;
        bool in = false;
        for (const ScanSpan &s : tr.spans[t]) in = in || (off >= 16 * s.lo && off + len <= 16 * s.hi);
        outside = outside || !in;
        max_read = std::max(max_read, len);
        memcpy(dst, tr.index[t].data() + off, len);
        return 0;
    };
    auto read_cut = [&](uint32_t c, uint64_t off, uint64_t len, void *dst) {
        if (off + len > cut_index[c].size()) return 5;
        memcpy(dst, cut_index[c].data() + off, len);
        return 0;
    };
    auto read_whole = [&](uint32_t t, uint64_t off, uint64_t len, void *dst) {
        if (off + len > tr.index[t].size()) return 5;
        memcpy(dst, tr.index[t].data() + off, len);
        return 0;
    };
    std::vector<std::vector<ScanSpan>> whole(n);
    for (uint32_t t = 0; t < n; t++) whole[t] = {ScanSpan{0, tr.ilen[t] / 16}};
    bool ok = true;
    for (int a = 2; a < argc && ok; a++) {
        const uint64_t budget = strtoull(argv[a], nullptr, 10);
        ScanPlan got, cut, want, full, full_spans;
        if (dbeel::plan_scan(tr.dlen.data(), tr.ilen.data(), n, budget, read, &got, &tr.spans)) return 4;
        if (dbeel::plan_scan(cdlen.data(), cilen.data(), (uint32_t)orig.size(), budget, read_cut, &cut)) return 4;
        if (dbeel::plan_scan(tr.dlen.data(), tr.ilen.data(), n, budget, read_whole, &full)) return 4;
        if (dbeel::plan_scan(tr.dlen.data(), tr.ilen.data(), n, budget, read_whole, &full_spans, &whole)) return 4;
        // map the cut plan back
        for (const dbeel::ScanPart &p : cut.parts) {
            dbeel::ScanPart q = p;
            q.first_slice = (uint32_t)want.slices.size();
            q.n_slices = 0;
            for (uint32_t k = 0; k < p.n_slices; k++) {
                const ScanSlice &s = cut.slices[p.first_slice + k];
                const uint32_t t = orig[s.table];
                for (uint64_t i = s.rec_lo; i < s.rec_hi; i++) {
                    const uint64_t r = map[s.table][i];
                    const uint8_t *ix = tr.index[t].data() + 16 * r;
                    const uint64_t lo = rd(ix, 8), hi = lo + rd(ix + 12, 4);
                    ScanSlice *last = q.n_slices ? &want.slices.back() : nullptr;
                    if (last && last->table == t && last->rec_hi == r) {
                        last->rec_hi = r + 1;
                        last->win_lo = std::min(last->win_lo, lo);
                        last->win_hi = std::max(last->win_hi, hi);
                    } else {
                        want.slices.push_back(ScanSlice{t, r, r + 1, lo, hi});
                        q.n_slices++;
                    }
                }
            }
            want.parts.push_back(q);
        }
        if (cut.panic_table >= 0) {
            const uint32_t c = (uint32_t)cut.panic_table;
            want.panic_table = (int32_t)orig[c];
            want.panic_record = map[c].empty() ? 0 : map[c][cut.panic_record];
        }
        ok = same_plan(got, want, "span plan vs cut plan", budget) && same_plan(full_spans, full, "whole spans vs no spans", budget);
    }
    if (ok && outside) {
        printf("the span plan read outside the spans\n");
        ok = false;
    }
    if (ok && max_read > dbeel::kScanPlanPiece) {
        printf("a read of %llu bytes\n", (unsigned long long)max_read);
        ok = false;
    }
    if (ok) printf("ok\n");
    return ok ? 0 : 1;
}

} // namespace

int main(int argc, char **argv) {
    if (argc >= 3 && !strcmp(argv[1], "spans")) return run_spans(argc, argv);
    fprintf(stderr, "usage: %s spans BUDGET... < tree\n", argv[0]);
    return 2;
}
