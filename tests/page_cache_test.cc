// Host checks of the readers' page cache policy in dbeel_b200/csrc/host/page_cache.h (driven by tests/test_page_cache_host.py).
//   check SEED  random request sequences over several tables whose files are not page multiples, carried out on a byte
//               model of the slots and the destination image: every range arrives with its file's bytes, every resident
//               page holds its file's bytes, reads cover exactly the missing pages as maximal page-aligned runs (ending on
//               a page boundary or at EOF) cut at the piece size, no resident page is read, the request's pages are never
//               evicted by it, resident <= capacity, the counters add up, every move is congruent modulo 16, and a failed
//               read inserts nothing
//   trace SEED  one JSON line per request (its parts, whether its reads succeeded, the pages it evicted, its hits and
//               misses) for the Python restatement of CLOCK to replay
// check prints "ok" or the first mismatch.
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <random>
#include <set>
#include <string>
#include <tuple>
#include <vector>

#include "../dbeel_b200/csrc/host/page_cache.h"

using namespace dbeel;

static uint8_t file_byte(uint64_t table, uint32_t kind, uint64_t off) {
    uint64_t h = (table * 1000003ull + kind * 7919ull + off) * 0x9E3779B97F4A7C15ull;
    return (uint8_t)(h >> 56);
}

struct Table { uint64_t id, len[3]; };

static std::vector<PagePart> random_request(std::mt19937_64 &rng, const std::vector<Table> &tabs, uint64_t *dst_end) {
    std::vector<PagePart> parts;
    const int np = 1 + (int)(rng() % 3);
    uint64_t pos = 0;
    for (int i = 0; i < np; i++) {
        const Table &t = tabs[rng() % tabs.size()];
        const uint32_t kind = 1 + (uint32_t)(rng() % 2);
        PagePart q{t.id, kind, t.len[kind], {}};
        const int nr = (int)(rng() % 5);
        for (int k = 0; k < nr && t.len[kind]; k++) {
            const uint64_t span = 1 + rng() % (rng() % 4 == 0 ? 40000 : 3000);
            const uint64_t lo = rng() % t.len[kind], hi = std::min(t.len[kind], lo + span);
            pos = (pos + 16 + 15) / 16 * 16 + (lo & 15); // as gvs_stage: congruent to the file offset modulo 16
            q.ranges.push_back(PageRange{lo, hi, pos});
            pos += hi - lo + 16;
        }
        parts.push_back(q);
    }
    *dst_end = pos + 16;
    return parts;
}

static int check(uint64_t seed) {
    std::mt19937_64 rng(seed);
    const uint64_t piece = 3 * kPageBytes; // small, so that runs are cut
    for (int round = 0; round < 40; round++) {
        std::vector<Table> tabs;
        const int nt = 1 + (int)(rng() % 4);
        for (int i = 0; i < nt; i++) {
            Table t{100 + (uint64_t)round * 10 + (uint64_t)i, {0, 0, 0}};
            for (int k = 1; k <= 2; k++) {
                const uint64_t c = rng() % 6;
                t.len[k] = c == 0 ? 1 + rng() % 4095 : c == 1 ? 16 * (1 + rng() % 200) : 1 + rng() % 200000; // shorter than one page, index-like, any
            }
            tabs.push_back(t);
        }
        const uint64_t cap = 1 + rng() % 48;
        PageCache pc(cap);
        std::vector<uint8_t> slots(cap * kPageBytes, 0); // the slots, one after the other as on the device
        std::map<std::tuple<uint64_t, uint32_t, uint64_t>, bool> resident; // the model's resident set
        uint64_t hits = 0, misses = 0, evictions = 0;
        for (int req = 0; req < 60; req++) {
            uint64_t dst_end = 0;
            const std::vector<PagePart> parts = random_request(rng, tabs, &dst_end);
            std::set<std::tuple<uint64_t, uint32_t, uint64_t>> want;
            for (const PagePart &q : parts)
                for (const PageRange &r : q.ranges)
                    for (uint64_t pg = r.lo / kPageBytes; pg <= (r.hi - 1) / kPageBytes; pg++) want.insert({q.table, q.kind, pg});
            const bool fail_reads = rng() % 7 == 0;
            PagePlan p = pc.plan(parts, piece);
            if (p.bypass) {
                if (want.size() <= cap) return printf("check: bypass of %zu pages with %llu slots\n", want.size(), (unsigned long long)cap), 1;
                if (pc.hits != hits || pc.misses != misses || pc.evictions != evictions) return printf("check: a bypass counted\n"), 1;
                continue;
            }
            if (want.size() > cap) return printf("check: %zu pages planned in %llu slots\n", want.size(), (unsigned long long)cap), 1;
            // pages read: exactly the missing ones, in maximal runs cut at the piece size
            std::set<std::tuple<uint64_t, uint32_t, uint64_t>> read_pages;
            std::vector<uint8_t> img(p.img_bytes + kPageBytes, 0xEE);
            for (size_t k = 0; k < p.reads.size(); k++) {
                const PageRead &rd = p.reads[k];
                const PagePart &q = parts[rd.part];
                if (rd.off % kPageBytes || rd.len == 0 || rd.len > piece || rd.img % 16) return printf("check: read %llu+%llu\n", (unsigned long long)rd.off, (unsigned long long)rd.len), 1;
                if (rd.off + rd.len > q.file_len) return printf("check: read past EOF\n"), 1;
                if ((rd.off + rd.len) % kPageBytes && rd.off + rd.len != q.file_len) return printf("check: read ends inside a page\n"), 1;
                const bool cont = k > 0 && p.reads[k - 1].part == rd.part && p.reads[k - 1].off + p.reads[k - 1].len == rd.off;
                if (cont && p.reads[k - 1].len != piece) return printf("check: a run cut below the piece size\n"), 1;
                if (cont && p.reads[k - 1].img + p.reads[k - 1].len != rd.img) return printf("check: a run not contiguous in the image\n"), 1;
                for (uint64_t o = rd.off; o < rd.off + rd.len; o += kPageBytes) {
                    const auto key = std::make_tuple(q.table, q.kind, o / kPageBytes);
                    if (resident.count(key)) return printf("check: a resident page is read\n"), 1;
                    if (!read_pages.insert(key).second) return printf("check: a page read twice in one request\n"), 1;
                }
                for (uint64_t b = 0; b < rd.len; b++) img[rd.img + b] = file_byte(q.table, q.kind, rd.off + b);
            }
            for (size_t k = 0; k < p.reads.size(); k++) // maximal: two runs of a part never touch
                for (size_t j = 0; j < p.reads.size(); j++)
                    if (j != k && p.reads[j].part == p.reads[k].part && p.reads[j].off == p.reads[k].off + p.reads[k].len &&
                        !(j == k + 1 && p.reads[k].len == piece))
                        return printf("check: adjacent missing pages in two runs\n"), 1;
            uint64_t n_miss = 0, n_hit = 0;
            for (const auto &key : want) (resident.count(key) ? n_hit : n_miss)++;
            if (read_pages.size() != n_miss || p.misses != n_miss || p.hits != n_hit) return printf("check: %zu pages read for %llu missing\n", read_pages.size(), (unsigned long long)n_miss), 1;
            for (const PageKey &k : p.evicted) {
                const auto key = std::make_tuple(k.table, k.kind, k.page);
                if (want.count(key)) return printf("check: a page of the request evicted\n"), 1;
                if (!resident.erase(key)) return printf("check: evicted a page not resident\n"), 1;
            }
            hits += n_hit;
            misses += n_miss;
            evictions += p.evicted.size();
            if (!fail_reads) { // carry the moves out: fills first (they come first), then the ranges
                std::vector<uint8_t> dst(dst_end, 0xDD);
                std::set<uint64_t> filled; // one launch runs every move at once: no move may read a slot a fill writes
                for (const PageMove &m : p.moves)
                    if (m.how == kPageImgToSlot) filled.insert(m.dst / kPageBytes);
                for (const PageMove &m : p.moves)
                    if (m.how == kPageSlotToDst)
                        for (uint64_t s = m.src / kPageBytes; s <= (m.src + m.len - 1) / kPageBytes; s++)
                            if (filled.count(s)) return printf("check: a hit read from a slot being filled\n"), 1;
                for (const PageMove &m : p.moves) {
                    if (m.how == kPageSlotToDst && m.src + m.len > slots.size()) return printf("check: a move past the slots\n"), 1;
                    const uint8_t *src = m.how == kPageSlotToDst ? &slots[m.src] : &img[m.src];
                    if (m.how == kPageImgToSlot && (m.dst % kPageBytes || m.len > kPageBytes)) return printf("check: a fill off its slot\n"), 1;
                    if ((m.src - m.dst) % 16) return printf("check: a move not congruent modulo 16\n"), 1;
                    uint8_t *d = m.how == kPageImgToSlot ? &slots[m.dst] : &dst[m.dst];
                    for (uint64_t b = 0; b < m.len; b++) d[b] = src[b];
                }
                for (const PagePart &q : parts)
                    for (const PageRange &r : q.ranges)
                        for (uint64_t o = r.lo; o < r.hi; o++)
                            if (dst[r.dst + o - r.lo] != file_byte(q.table, q.kind, o)) return printf("check: range byte %llu wrong\n", (unsigned long long)o), 1;
                for (const auto &key : read_pages) resident[key] = true;
            }
            pc.commit(p, !fail_reads);
            if (pc.resident() != resident.size() || pc.resident() > cap) return printf("check: %llu resident, model %zu, capacity %llu\n", (unsigned long long)pc.resident(), resident.size(), (unsigned long long)cap), 1;
            for (const auto &kv : resident)
                if (!pc.holds(PageKey{std::get<0>(kv.first), std::get<1>(kv.first), std::get<2>(kv.first)})) return printf("check: resident sets differ\n"), 1;
            if (pc.hits != hits || pc.misses != misses || pc.evictions != evictions) return printf("check: counters\n"), 1;
        }
        // every resident page holds its file's bytes: plan a request of all of them, all hits, and read the slots
        std::vector<PagePart> all;
        for (const auto &kv : resident) {
            const Table *t = nullptr;
            for (const Table &x : tabs) if (x.id == std::get<0>(kv.first)) t = &x;
            const uint32_t kind = std::get<1>(kv.first);
            const uint64_t lo = std::get<2>(kv.first) * kPageBytes, hi = std::min(t->len[kind], lo + kPageBytes);
            all.push_back(PagePart{t->id, kind, t->len[kind], {PageRange{lo, hi, 0}}});
        }
        PagePlan p = pc.plan(all, piece);
        if (p.misses || !p.reads.empty()) return printf("check: a resident page missed\n"), 1;
        if (p.moves.size() != all.size()) return printf("check: %zu moves for %zu resident pages\n", p.moves.size(), all.size()), 1;
        for (size_t i = 0; i < all.size(); i++) {
            const PageMove &m = p.moves[i];
            const PagePart &q = all[i];
            if (m.len != q.ranges[0].hi - q.ranges[0].lo) return printf("check: whole-page move of %llu bytes\n", (unsigned long long)m.len), 1;
            for (uint64_t b = 0; b < m.len; b++)
                if (slots[m.src + b] != file_byte(q.table, q.kind, q.ranges[0].lo + b)) return printf("check: a slot holds wrong bytes\n"), 1;
        }
        pc.commit(p, true);
    }
    printf("ok\n");
    return 0;
}

static int trace(uint64_t seed) {
    std::mt19937_64 rng(seed);
    std::vector<Table> tabs;
    for (int i = 0; i < 3; i++) tabs.push_back(Table{7 + (uint64_t)i, {0, 1 + rng() % 60000, 16 * (1 + rng() % 2000)}});
    const uint64_t cap = 4 + rng() % 24;
    PageCache pc(cap);
    printf("{\"capacity\": %llu}\n", (unsigned long long)cap);
    for (int req = 0; req < 300; req++) {
        uint64_t dst_end;
        const std::vector<PagePart> parts = random_request(rng, tabs, &dst_end);
        const bool ok = rng() % 9 != 0;
        PagePlan p = pc.plan(parts, 8 * kPageBytes);
        printf("{\"parts\": [");
        for (size_t i = 0; i < parts.size(); i++) {
            printf("%s[%llu, %u, %llu, [", i ? ", " : "", (unsigned long long)parts[i].table, parts[i].kind, (unsigned long long)parts[i].file_len);
            for (size_t k = 0; k < parts[i].ranges.size(); k++)
                printf("%s[%llu, %llu]", k ? ", " : "", (unsigned long long)parts[i].ranges[k].lo, (unsigned long long)parts[i].ranges[k].hi);
            printf("]]");
        }
        printf("], \"ok\": %s, \"bypass\": %s, \"hits\": %llu, \"misses\": %llu, \"evicted\": [", ok ? "true" : "false",
               p.bypass ? "true" : "false", (unsigned long long)p.hits, (unsigned long long)p.misses);
        for (size_t k = 0; k < p.evicted.size(); k++)
            printf("%s[%llu, %u, %llu]", k ? ", " : "", (unsigned long long)p.evicted[k].table, p.evicted[k].kind, (unsigned long long)p.evicted[k].page);
        printf("]}\n");
        if (!p.bypass) pc.commit(p, ok);
    }
    return 0;
}

int main(int argc, char **argv) {
    if (argc < 3) return 2;
    const std::string what = argv[1];
    const uint64_t seed = strtoull(argv[2], nullptr, 10);
    if (what == "check") return check(seed);
    if (what == "trace") return trace(seed);
    return 2;
}
