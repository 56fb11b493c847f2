// scan_seek.cuh -- dbeel_reader_scan's bound search: for every table and every bound of a key range, the first record whose
// key is not less than the bound (seek_t in dbeel_compact.h: lookup.cuh's exact-mode search with no exit on equality, so a
// comparison c == 0 goes to child 2k of the probe tree and the reader's DBEEL_LOOKUP_EXACT fences serve it as they are).
// Tables are independent and there is no filter, so every (table, bound) pair searches in one pass:
//
//   k_seek_fence  one thread per pair: descends the table's fences (GvsFences, the reader's cached ones or fences read for
//                 this call); finishes, fails at a corrupt fence (ffr == 0), or ends in a leaf it marks touched
//   k_seek_leaf   resumes inside the staged leaves (GvsLeaf: the table's TableDesc with .index / .data biased to the leaf's
//                 slice and window, so probe() checks the same bounds against the file's data_len) and finishes or fails
//
// A failed search leaves the probed record and its index record: the host turns the smallest failing record of a table into
// the scan's stop.
#pragma once

#include "lookup_stream.cuh"

namespace dbeel {

struct SeekQueries {
    const uint8_t *keys;          // the range keys
    const uint64_t *key_off;      // [n] bound key of pair q: keys[key_off[q] .. + key_len[q])
    const uint64_t *key_len;
    const uint32_t *table;        // [n] table of pair q
    uint64_t n;
    SearchState *state;           // the open search after the fences
    uint32_t *node;               // 0 = finished or failed, else its leaf node 2^depth + leaf
    unsigned long long *result;   // seek_t(bound) when it finished, else ~0
    unsigned long long *bad_rec;  // the record a probe reported corrupt, else ~0
    uint4 *bad_ix;                // its index record
};

__device__ __forceinline__ void seek_fail(const SeekQueries &g, uint64_t q, uint64_t pos, const uint4 &ix) {
    g.bad_rec[q] = pos;
    g.bad_ix[q] = ix;
}

// fences[t]: table t's fences; GvsFences.touched = the table's own leaf flags
__global__ void __launch_bounds__(256) k_seek_fence(SeekQueries g, const GvsFences *fences) {
    pdl_trigger();
    pdl_wait();
    const uint64_t q = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    if (q >= g.n) return;
    const GvsFences f = fences[g.table[q]];
    const uint8_t *key = g.keys + g.key_off[q];
    const uint64_t klen = g.key_len[q];
    SearchState s = search_init(1, f.n);
    uint32_t node = 1;
    g.result[q] = ~0ull;
    g.bad_rec[q] = ~0ull;
    const uint32_t leaf0 = 1u << f.depth;
    while (node < leaf0) {
        const unsigned long long fr = f.ffr[node];
        const uint64_t pos = search_pos(1, s);
        if (fr == 0) { // as probe(): offset or length prefix past the end of .data
            seek_fail(g, q, pos, f.fix[node]);
            node = 0;
            break;
        }
        const uint8_t *frame = reinterpret_cast<const uint8_t *>(fr);
        const int c = cmp_key_bytes(frame + 8, ld_bytes_le<true>(frame, 8), key, klen);
        search_step(1, f.n, &s, c);
        if (s.done) {
            g.result[q] = s.a;
            node = 0;
            break;
        }
        node = 2 * node + (c < 0 ? 1u : 0u);
    }
    g.node[q] = node;
    if (node) {
        g.state[q] = s;
        f.touched[node - leaf0] = 1;
    }
}

// The staged leaves of one group, ascending (table, leaf); table t's are leaves[first[t] .. first[t + 1]).  tables[t] is
// the table's TableDesc (data_len, n), depth[t] its fence depth.
__global__ void __launch_bounds__(256) k_seek_leaf(SeekQueries g, const TableDesc *tables, const uint32_t *depth,
                                                   const GvsLeaf *leaves, const uint32_t *first) {
    pdl_trigger();
    pdl_wait();
    const uint64_t q = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    if (q >= g.n) return;
    const uint32_t node = g.node[q];
    if (node == 0) return;
    const uint32_t ti = g.table[q], leaf = node - (1u << depth[ti]);
    uint32_t lo = first[ti], hi = first[ti + 1]; // the group's leaf, if it holds it
    while (lo < hi) {
        const uint32_t mid = (lo + hi) / 2;
        if (leaves[mid].leaf < leaf) lo = mid + 1; else hi = mid;
    }
    if (lo == first[ti + 1] || leaves[lo].leaf != leaf) return;
    TableDesc t = tables[ti];
    t.data = leaves[lo].data;
    t.index = leaves[lo].index;
    const uint8_t *key = g.keys + g.key_off[q];
    const uint64_t klen = g.key_len[q];
    SearchState s = g.state[q];
    while (!s.done) {
        uint4 ix;
        bool bad = false;
        const uint64_t pos = search_pos(1, s);
        const int c = probe(t, pos, key, klen, &bad, &ix);
        if (bad) {
            seek_fail(g, q, pos, ix);
            break;
        }
        search_step(1, t.n, &s, c);
    }
    if (s.done) g.result[q] = s.a;
    g.node[q] = 0;
}

} // namespace dbeel
