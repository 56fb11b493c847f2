// page_cache.h -- the policy of the readers' device page cache (dbeel_page_cache, dbeel_compact.h), in plain C++ so that
// tests/page_cache_test.cc can drive it without a GPU.  dbeel_compact.cu owns the slots (one device allocation) and carries
// out the plans made here; every decision about pages is made here and nowhere else.
//
// A page is kPageBytes bytes at a page-aligned offset of one table's .data or .index, keyed by (table id, file kind, page
// number).  A file's last page holds only the bytes up to the file's length.  Table ids are never reused, so the pages of
// a table that is gone are never hit again and age out.
//
// A request is a list of parts, one (table id, kind, file length, byte ranges) each, every range wanted at a position of
// one destination image.  Its plan:
//   reads   the missing pages, as page-aligned file ranges clipped to the file's length: consecutive missing pages of a
//           part are one run, cut into pieces of at most `piece` bytes, laid out one after the other in a miss image
//   moves   miss image -> slot (the fills), then per range its bytes from a slot (hits) or from the miss image (misses)
//           into the destination image; every move keeps its source and destination congruent modulo 16 as long as the
//           destination image places each range congruent to its file offset
//   evicted the pages that left the cache to make room, in order
// Eviction is CLOCK (second chance): a page's reference bit is set when it is inserted and when it is hit; the hand
// clears set bits and takes the first slot that is free or has its bit clear.  The pages of a request (hits and the
// slots taken for its misses) are pinned from plan() to commit(), so the request never evicts what it reads.  A missing
// page becomes resident only at commit(ok = true), after its read has succeeded; commit(ok = false) frees the slots taken
// for the misses and leaves every other page as it was.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <unordered_map>
#include <vector>

namespace dbeel {

constexpr uint64_t kPageBytes = 4096;

struct PageKey {
    uint64_t table;
    uint32_t kind;
    uint64_t page;
    bool operator==(const PageKey &o) const { return table == o.table && kind == o.kind && page == o.page; }
};

struct PageKeyHash {
    size_t operator()(const PageKey &k) const {
        uint64_t h = k.table * 0x9E3779B97F4A7C15ull ^ (k.page + 0x632BE59BD9B4E019ull) * 0xC2B2AE3D27D4EB4Full ^ k.kind;
        return (size_t)(h ^ (h >> 29));
    }
};

struct PageRange { uint64_t lo, hi, dst; }; // file bytes [lo, hi) wanted at dst of the destination image

struct PagePart {
    uint64_t table;
    uint32_t kind;
    uint64_t file_len;
    std::vector<PageRange> ranges;
};

struct PageRead { uint32_t part; uint64_t off, len, img; }; // file bytes [off, off + len) of the part's file -> miss image + img

enum : uint32_t { kPageImgToSlot = 0, kPageImgToDst = 1, kPageSlotToDst = 2 };

// src / dst: byte offsets into the miss image, the slots (slot * kPageBytes + offset) or the destination image, by `how`
struct PageMove { uint32_t how; uint64_t src, dst, len; };

struct PagePlan {
    bool bypass = false; // more distinct pages than slots, or a range outside its file: nothing planned, read uncached
    std::vector<PageRead> reads;
    std::vector<PageMove> moves;
    std::vector<PageKey> evicted;
    std::vector<std::pair<PageKey, uint32_t>> fresh; // the missing pages and their slots, resident after commit(ok)
    std::vector<uint32_t> pinned;
    uint64_t img_bytes = 0, hits = 0, misses = 0;
};

class PageCache {
  public:
    explicit PageCache(uint64_t slots) : slot_(slots) {}

    uint64_t capacity() const { return slot_.size(); }
    uint64_t resident() const { return map_.size(); }
    bool holds(const PageKey &k) const { return map_.count(k) != 0; }
    uint64_t hits = 0, misses = 0, evictions = 0; // pages, since creation

    PagePlan plan(const std::vector<PagePart> &parts, uint64_t piece) {
        PagePlan p;
        // where each distinct page of the request comes from: its slot (hit) or its place in the miss image (miss)
        struct Src { bool hit; uint64_t at; };
        std::unordered_map<PageKey, Src, PageKeyHash> src;
        for (const PagePart &q : parts)
            for (const PageRange &r : q.ranges) {
                if (r.lo > r.hi || r.hi > q.file_len) { p.bypass = true; return p; }
                for (uint64_t pg = r.lo / kPageBytes; r.lo < r.hi && pg <= (r.hi - 1) / kPageBytes; pg++)
                    src.emplace(PageKey{q.table, q.kind, pg}, Src{false, 0});
            }
        if (src.size() > slot_.size()) { p.bypass = true; return p; }
        // hits first, so that the misses' victims never take a page the request reads
        std::vector<std::vector<uint64_t>> miss(parts.size());
        for (size_t i = 0; i < parts.size(); i++) {
            const PagePart &q = parts[i];
            std::vector<uint64_t> pages;
            for (const PageRange &r : q.ranges)
                for (uint64_t pg = r.lo / kPageBytes; r.lo < r.hi && pg <= (r.hi - 1) / kPageBytes; pg++) pages.push_back(pg);
            std::sort(pages.begin(), pages.end());
            pages.erase(std::unique(pages.begin(), pages.end()), pages.end());
            for (uint64_t pg : pages) {
                const PageKey k{q.table, q.kind, pg};
                Src &s = src[k];
                if (s.hit || s.at) continue; // met in an earlier part of the request
                auto it = map_.find(k);
                if (it != map_.end()) {
                    Slot &x = slot_[it->second];
                    x.ref = true;
                    x.pinned = true;
                    p.pinned.push_back(it->second);
                    s = Src{true, it->second};
                    p.hits++;
                } else {
                    s.at = ~0ull; // claimed by this part
                    miss[i].push_back(pg);
                }
            }
        }
        for (size_t i = 0; i < parts.size(); i++) {
            const PagePart &q = parts[i];
            for (size_t a = 0, b; a < miss[i].size(); a = b) {
                for (b = a + 1; b < miss[i].size() && miss[i][b] == miss[i][b - 1] + 1; b++) {}
                const uint64_t lo = miss[i][a] * kPageBytes, hi = std::min(q.file_len, (miss[i][b - 1] + 1) * kPageBytes);
                const uint64_t img = (p.img_bytes + 15) / 16 * 16;
                for (uint64_t d = 0; d < hi - lo; d += piece) p.reads.push_back(PageRead{(uint32_t)i, lo + d, std::min(piece, hi - lo - d), img + d});
                p.img_bytes = img + (hi - lo);
                for (size_t j = a; j < b; j++) {
                    const PageKey k{q.table, q.kind, miss[i][j]};
                    const uint32_t s = victim(&p);
                    slot_[s].pinned = true;
                    p.pinned.push_back(s);
                    p.fresh.push_back({k, s});
                    const uint64_t at = img + (j - a) * kPageBytes;
                    src[k] = Src{false, at};
                    p.moves.push_back(PageMove{kPageImgToSlot, at, (uint64_t)s * kPageBytes, std::min(kPageBytes, q.file_len - miss[i][j] * kPageBytes)});
                    p.misses++;
                }
            }
        }
        // each range from its pages; a move that continues the previous one extends it
        for (const PagePart &q : parts)
            for (const PageRange &r : q.ranges)
                for (uint64_t x = r.lo; x < r.hi;) {
                    const uint64_t pg = x / kPageBytes, end = std::min(r.hi, (pg + 1) * kPageBytes);
                    const Src &s = src[PageKey{q.table, q.kind, pg}];
                    const PageMove m{s.hit ? kPageSlotToDst : kPageImgToDst, (s.hit ? s.at * kPageBytes : s.at) + (x - pg * kPageBytes),
                                     r.dst + (x - r.lo), end - x};
                    PageMove *l = p.moves.empty() ? nullptr : &p.moves.back();
                    if (l && l->how == m.how && l->src + l->len == m.src && l->dst + l->len == m.dst) l->len += m.len;
                    else p.moves.push_back(m);
                    x = end;
                }
        hits += p.hits;
        misses += p.misses;
        return p;
    }

    // ok: every read of the plan returned 0 (its missing pages become resident); else the slots taken for them are freed
    void commit(PagePlan &p, bool ok) {
        for (const auto &f : p.fresh) {
            Slot &x = slot_[f.second];
            if (ok) {
                x.key = f.first;
                x.used = true;
                x.ref = true;
                map_[f.first] = f.second;
            }
        }
        for (uint32_t s : p.pinned) slot_[s].pinned = false;
        p.fresh.clear();
        p.pinned.clear();
    }

  private:
    struct Slot {
        PageKey key{0, 0, 0};
        bool used = false, ref = false, pinned = false;
    };
    std::vector<Slot> slot_;
    std::unordered_map<PageKey, uint32_t, PageKeyHash> map_;
    uint64_t hand_ = 0;

    // the CLOCK hand's next slot: free, or holding a page whose reference bit is clear (evicted); pinned slots are passed
    // over.  plan() pins at most capacity() slots, so one is always found within two turns.
    uint32_t victim(PagePlan *p) {
        for (;;) {
            const uint32_t s = (uint32_t)hand_;
            hand_ = (hand_ + 1) % slot_.size();
            Slot &x = slot_[s];
            if (x.pinned) continue;
            if (!x.used) return s;
            if (x.ref) { x.ref = false; continue; }
            map_.erase(x.key);
            x.used = false;
            evictions++;
            p->evicted.push_back(x.key);
            return s;
        }
    }
};

} // namespace dbeel
