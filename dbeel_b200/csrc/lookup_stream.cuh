// lookup_stream.cuh -- dbeel_get_values_stream: the search of lookup.cuh on tables that are not on the device, only the parts
// of them the batch's searches reach (host/lookup_plan.h).  Per table, newest first, for the queries still open:
//
//   k_gvs_filter   the table's bloom filter; an open query that passes starts its search at the root (node 1)
//   k_lookup_fence the top D probes on the staged fences (index record + key frame per probe-tree node); ends in a hit, a
//                  corrupt record, "not in this table", or a leaf (node 2^D + leaf) whose records are staged next
//   k_lookup_leaf  resumes the search inside a staged leaf: the table's TableDesc with .index / .data biased to the slice and
//                  the window, so probe() checks the same bounds against the file's data_len as k_lookup does
//   k_gvs_copy     copies the entries of the group's hits out of the window into the hit heap before the window is reused
//
// Hits at fences have no window: their entries are read one record each after the last table.  Then k_gvs_hit decodes
// every hit's entry from the heap the way k_lookup_emit decodes it.
// Per query: its row (dbeel_lookup_result), the hit's index record, its search state and node, and where its entry is.
#pragma once

#include "lookup.cuh"
#include "host/lookup_plan.h"

namespace dbeel {

struct GvsQueries {
    const uint8_t *keys;
    const uint64_t *key_off;
    uint64_t n_keys;
    uint4 *rows;          // {table, rejects | flags, record lo, record hi}; table = ~0 while not found
    uint4 *hit_ix;        // the hit's index record
    SearchState *state;   // the search in the current table
    uint32_t *node;       // 0 = nothing to do in the current table, else its probe-tree node
    unsigned long long *hit_src; // a leaf hit's entry inside the staged window, until k_gvs_copy has copied it (else 0)
    unsigned long long *hit_off; // the entry's offset in the hit heap, kGvsNoEntry or kGvsFenceHit
    uint32_t mode;
};

constexpr unsigned long long kGvsNoEntry = ~0ull;      // no hit, or a hit whose entry cannot decode
constexpr unsigned long long kGvsFenceHit = ~0ull - 1; // a hit at a fence: its entry is read after the last table

// The index-level half of k_lookup_emit's decode: key_size == 8 + klen, room for the value frame and the timestamp, the
// entry inside .data (off <= data_len).  Only entries that pass it are copied or read.
__host__ __device__ __forceinline__ bool gvs_entry_fits(uint64_t off, uint64_t ks, uint64_t fs, uint64_t klen, uint64_t data_len) {
    return ks == 8 + klen && fs >= ks + 24 && off <= data_len && fs <= data_len - off;
}

__device__ __forceinline__ bool gvs_closed(const uint4 &r) { return r.x != 0xFFFFFFFFu || (r.y & kLookupCorrupt); }

__global__ void __launch_bounds__(256) k_gvs_filter(GvsQueries g, TableDesc t, unsigned long long *n_open) {
    pdl_trigger();
    pdl_wait();
    const uint64_t q = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    if (q >= g.n_keys) return;
    g.node[q] = 0;
    uint4 r = g.rows[q];
    if (gvs_closed(r)) return;
    const uint64_t k0 = g.key_off[q];
    const uint8_t *key = g.keys + k0;
    const uint64_t klen = g.key_off[q + 1] - k0;
    if (t.words != nullptr) { // as lookup_query
        uint64_t h0, h1;
        sip13_pair_vec_u8(t.sip, klen, [key, klen](uint64_t w) {
            const uint64_t left = klen - 8 * w;
            return ld_bytes_le<false>(key + 8 * w, left < 8 ? (uint32_t)left : 8u);
        }, &h0, &h1);
        bool all = true;
        const uint32_t *words = t.words;
        bloom_probe_all(h0, h1, t.k_num, t.bits, t.bits_magic,
                        [&all, words](uint64_t bit) { all = all && ((__ldg(&words[bit >> 5]) >> (bit & 31)) & 1u); });
        if (!all) {
            r.y++;
            g.rows[q] = r;
            return;
        }
    }
    if (t.n == 0) return;
    g.state[q] = search_init(g.mode, t.n);
    g.node[q] = 1;
    atomicAdd(n_open, 1ull);
}

// fences: per node k < 2^depth the index record fix[k] and the device address of its key frame ffr[k] (0 = the probe
// reports the record corrupt); touched[leaf] is set for every leaf a search ends in.
struct GvsFences {
    const uint4 *fix;
    const unsigned long long *ffr;
    uint32_t depth;
    uint32_t table;
    uint64_t n;
    uint8_t *touched;
};

__global__ void __launch_bounds__(256) k_lookup_fence(GvsQueries g, GvsFences f) {
    pdl_trigger();
    pdl_wait();
    const uint64_t q = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    if (q >= g.n_keys) return;
    uint32_t node = g.node[q];
    if (node == 0) return;
    const uint64_t k0 = g.key_off[q];
    const uint8_t *key = g.keys + k0;
    const uint64_t klen = g.key_off[q + 1] - k0;
    SearchState s = g.state[q];
    const uint32_t leaf0 = 1u << f.depth;
    while (node < leaf0) {
        const unsigned long long fr = f.ffr[node];
        const uint64_t pos = search_pos(g.mode, s);
        if (fr == 0) { // as probe(): offset or length prefix past the end of .data
            g.rows[q].y |= kLookupCorrupt;
            node = 0;
            break;
        }
        const uint8_t *frame = reinterpret_cast<const uint8_t *>(fr);
        const int c = cmp_key_bytes(frame + 8, ld_bytes_le<true>(frame, 8), key, klen);
        if (c == 0) {
            const uint4 r = g.rows[q];
            g.rows[q] = make_uint4(f.table, r.y, (uint32_t)pos, (uint32_t)(pos >> 32));
            g.hit_ix[q] = f.fix[node];
            g.hit_off[q] = kGvsFenceHit;
            node = 0;
            break;
        }
        search_step(g.mode, f.n, &s, c);
        if (s.done) { node = 0; break; }
        node = 2 * node + (c < 0 ? 1u : 0u);
    }
    g.node[q] = node;
    if (node) {
        g.state[q] = s;
        f.touched[node - leaf0] = 1;
    }
}

// The staged leaves of one group, ascending leaf ids; data / index are biased so that file offset o / record r of the table
// are at data + o / index + r.
struct GvsLeaf {
    const uint8_t *data;
    const uint4 *index;
    uint32_t leaf, pad;
    uint64_t pad2;
};

// A hit whose entry fits (gvs_entry_fits) leaves its window address in hit_src and adds the heap bytes k_gvs_copy will
// take for it to *heap_need.
__global__ void __launch_bounds__(256) k_lookup_leaf(GvsQueries g, TableDesc t, const GvsLeaf *leaves, uint32_t n_leaves,
                                                     uint32_t depth, uint32_t table, unsigned long long *heap_need) {
    pdl_trigger();
    pdl_wait();
    const uint64_t q = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    if (q >= g.n_keys) return;
    const uint32_t node = g.node[q], leaf0 = 1u << depth;
    if (node < leaf0) return;
    const uint32_t leaf = node - leaf0;
    uint32_t lo = 0, hi = n_leaves; // the group's leaf, if it holds it
    while (lo < hi) {
        const uint32_t mid = (lo + hi) / 2;
        if (leaves[mid].leaf < leaf) lo = mid + 1; else hi = mid;
    }
    if (lo == n_leaves || leaves[lo].leaf != leaf) return;
    t.data = leaves[lo].data;
    t.index = leaves[lo].index;
    const uint64_t k0 = g.key_off[q];
    const uint8_t *key = g.keys + k0;
    const uint64_t klen = g.key_off[q + 1] - k0;
    SearchState s = g.state[q];
    bool bad = false;
    while (!s.done) {
        uint4 ix;
        const uint64_t pos = search_pos(g.mode, s);
        const int c = probe(t, pos, key, klen, &bad, &ix);
        if (bad) {
            g.rows[q].y |= kLookupCorrupt;
            break;
        }
        if (c == 0) {
            const uint4 r = g.rows[q];
            g.rows[q] = make_uint4(table, r.y, (uint32_t)pos, (uint32_t)(pos >> 32));
            g.hit_ix[q] = ix;
            const uint64_t off = (uint64_t)ix.x | ((uint64_t)ix.y << 32), fs = ix.w;
            if (gvs_entry_fits(off, ix.z, fs, klen, t.data_len)) { // the window covers [off, off + fs) (lookup_plan.h)
                g.hit_src[q] = reinterpret_cast<unsigned long long>(t.data + off);
                atomicAdd(heap_need, (unsigned long long)((fs + 15) / 16 * 16 + 16));
            }
            break;
        }
        search_step(g.mode, t.n, &s, c);
    }
    g.node[q] = 0;
}

// One warp per query: a leaf hit's entry from its window into the hit heap, at a position congruent to the source modulo
// 16 (16-byte copies in the middle, bytes at the ends), so entries of any size, multi-megabyte ones included, move at once.
__global__ void __launch_bounds__(256) k_gvs_copy(GvsQueries g, uint8_t *heap, unsigned long long *cursor) {
    pdl_trigger();
    pdl_wait();
    const uint64_t q = ((uint64_t)blockIdx.x * 256u + threadIdx.x) / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (q >= g.n_keys) return;
    const unsigned long long src = g.hit_src[q];
    if (src == 0) return;
    const uint64_t fs = g.hit_ix[q].w;
    unsigned long long pos = 0;
    if (lane == 0) pos = atomicAdd(cursor, (unsigned long long)((fs + 15) / 16 * 16 + 16));
    pos = __shfl_sync(0xFFFFFFFFu, pos, 0) + (src & 15);
    const uint8_t *s = reinterpret_cast<const uint8_t *>(src);
    uint8_t *d = heap + pos;
    const uint64_t head = ((16 - (src & 15)) & 15) < fs ? ((16 - (src & 15)) & 15) : fs;
    const uint64_t body = (fs - head) / 16, tail0 = head + 16 * body;
    for (uint64_t i = lane; i < head; i += 32) d[i] = s[i];
    for (uint64_t i = lane; i < body; i += 32) reinterpret_cast<uint4 *>(d + head)[i] = reinterpret_cast<const uint4 *>(s + head)[i];
    for (uint64_t i = tail0 + lane; i < fs; i += 32) d[i] = s[i];
    if (lane == 0) {
        g.hit_off[q] = pos;
        g.hit_src[q] = 0;
    }
}

// After the last table: every hit's entry as k_lookup_emit decodes it, from the heap (hit_off: its offset there, or
// kGvsNoEntry / kGvsFenceHit when it was not copied or read because it cannot decode).
__global__ void __launch_bounds__(256) k_gvs_hit(GvsQueries g, const uint8_t *heap, LookupEmit em) {
    pdl_trigger();
    pdl_wait();
    const uint64_t q = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    if (q >= g.n_keys) return;
    uint4 r = g.rows[q];
    uint32_t d = kScanNone;
    uint4 rec = make_uint4(0, 0, 0, 0);
    if (r.x != 0xFFFFFFFFu) {
        const uint64_t klen = g.key_off[q + 1] - g.key_off[q];
        const uint4 ix = g.hit_ix[q];
        const uint64_t ks = ix.z, fs = ix.w;
        const unsigned long long ho = g.hit_off[q];
        const unsigned long long a = ho >= kGvsFenceHit ? 0ull : reinterpret_cast<unsigned long long>(heap + ho);
        bool ok = a != 0 && ks == 8 + klen && fs >= ks + 24;
        if (ok) {
            const uint8_t *e = reinterpret_cast<const uint8_t *>(a);
            ok = ld_bytes_le<true>(e + ks, 8) == fs - ks - 24 && ts_decodes(ld_bytes_le<true>(e + fs - 16, 8), ld_bytes_le<true>(e + fs - 8, 8));
        }
        if (ok) {
            d = 0;
            rec = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)ks, (uint32_t)fs);
        } else {
            r.y |= kLookupBadEntry;
            g.rows[q] = r;
        }
    }
    em.dest[q] = d;
    em.flat[q] = rec;
}

} // namespace dbeel
