// range_limit.cuh -- one merge round of dbeel_reader_get_ranges / _reverse / dbeel_readers_get_ranges: per query, a
// prefix (forward) or a suffix (reverse, LimitQuery.desc) of every table's span records (a "pair" = one query and one table, its chunk staged as
// {entry address, index status, full_size} records), merged into the query's first (forward) or last (reverse) entries
// under dbeel_reader_get_range's rule -- the newest table's version of a key wins, tombstones dropped unless asked for.
// Direction and the tombstone rule are the query's own, so one round serves forward and reverse queries of many readers.
// Pairs of a query lie together, tables ascending; a pair's records lie in record order in both directions.
//
//   k_limit_decode  per record: the scan's decode (PANIC / ERR), the flat split record {address, 8 + klen, full_size},
//                   the big-endian 8-byte key prefix, and strict ascent over the pair's neighbour record -- forward the
//                   previous one (a violation flags the higher record), reverse the next one (it flags the lower); per
//                   pair the damaged record met first from the chunk's fixed end (atomicMin of its distance from there)
//   k_limit_query   per query: the first damaged pair, else the frontier F_q over the pairs whose chunk stopped short of
//                   the span's far end -- forward the smallest last staged key (every key <= F_q is complete), reverse
//                   the largest first staged key (every key >= F_q is) -- and the pairs that set it
//   k_limit_flag    per record: keep = the query is clean, key on the complete side of F_q, no newer pair staged the key,
//                   tombstone rule
//   k_range_tile_sums / k_range_tile_scan / k_range_prefix (merge_range.cuh) on one segment: exclusive prefix sum of keep
//   k_limit_rank    per survivor: its merged position in the query's output order (own pair's survivors before it --
//                   after it, reverse -- + every other pair's survivors below its key -- above it, reverse); per query:
//                   its survivors
//   k_limit_select  per survivor of a finished query with rank < limit: its split record to out slot base + rank
// The selected records then go through the split and phase 2 (split_emit) unchanged, in rank order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "device_fns.cuh"
#include "merge_range.cuh"
#include "scan.cuh"

namespace dbeel {

constexpr uint32_t kLimitUnsorted = 4u; // damage code of a record not above its predecessor (after kScanStopErr / Panic)

struct LimitPair {
    uint32_t first, count; // its records [first, first + count) of the round
    uint32_t query, truncated; // truncated: the chunk stopped short of the span's far end (its end; reverse: its start)
};

struct LimitQuery {
    uint32_t pair0, pair1; // its pairs
    uint32_t first, last;  // its records
    uint32_t limit;
    uint16_t desc;            // 1: reverse -- chunks end at the span's end, the last entries in descending key order
    uint16_t keep_tombstones; // 1: tombstones are entries
};

struct LimitParams {
    const LimitPair *pairs;
    const LimitQuery *queries;
    const uint4 *rec;              // [n] {entry address (x, y), kScanStopPanic when the index record alone shows it, full_size}
    const uint32_t *rpair;         // [n] pair of every record
    uint32_t n, n_queries;
    uint4 *flat;                   // [n] {entry address, 8 + klen, full_size}
    unsigned long long *pfx;       // [n]
    uint32_t *code;                // [n] 0 or the record's damage (kScanStopErr, kScanStopPanic, kLimitUnsorted)
    uint32_t *pair_bad;            // [pairs] the pair's damaged record nearest its chunk's fixed end, as its distance from
                                   // there (forward: from the first record, reverse: from the last), ~0 = none
    uint32_t *setter;              // [pairs] 1: the pair's last (reverse: first) staged key is F_q
    uint32_t *front;               // [queries] the record that holds F_q, ~0 = every pair read to its span's end
    uint4 *qout;                   // [queries] {survivors on F_q's complete side, damage code, damaged pair, its pair_bad}
    const uint32_t *pre;           // [n + 1] keep, then its exclusive prefix sum (k_range_prefix)
    uint32_t *keep;                // the same array, written by k_limit_flag
    uint32_t *rank;                // [n]
    const uint32_t *qsel;          // [queries] out slot of a finished query's first entry, ~0 = not finished this round
    uint4 *sel_flat;               // ScanParams.flat / .dest of the split
    uint32_t *sel_dest;
};

// bincode Entry from exactly fs bytes at e (k_scan_classify's checks): *klen on success
__device__ __forceinline__ bool limit_decode(const uint4 &r, uint64_t *klen) {
    if (r.z) return false;
    const uint8_t *e = reinterpret_cast<const uint8_t *>((uint64_t)r.x | ((uint64_t)r.y << 32));
    const uint64_t fs = r.w;
    if (fs < 8) return false;
    const uint64_t kl = ld_u64_unaligned_narrow(e);
    if (kl > fs - 8 || fs - 8 - kl < 8) return false;
    const uint64_t dlen = ld_u64_unaligned_narrow(e + 8 + kl), rest = fs - 16 - kl;
    if (dlen > rest || rest - dlen != 16) return false;
    if (!ts_decodes(ld_u64_unaligned_narrow(e + fs - 16), ld_u64_unaligned_narrow(e + fs - 8))) return false;
    *klen = kl;
    return true;
}

// Vec<u8>::cmp of the keys of decoded records i and j
__device__ __forceinline__ int limit_cmp(const LimitParams &p, uint32_t i, unsigned long long pi, const uint8_t *k, uint32_t kl,
                                         uint32_t j) {
    const unsigned long long pj = p.pfx[j];
    if (pj != pi) return pj < pi ? 1 : -1;
    const uint4 r = p.flat[j];
    return -scan_key_cmp(range_entry(r) + 8, r.z - 8, k, kl);
}

// first record of pair pp whose key is >= k
__device__ __forceinline__ uint32_t limit_lower_bound(const LimitParams &p, const LimitPair &pp, unsigned long long pk, const uint8_t *k,
                                                      uint32_t kl) {
    uint32_t a = pp.first, b = pp.first + pp.count;
    while (a < b) {
        const uint32_t mid = a + ((b - a) >> 1);
        if (limit_cmp(p, 0, pk, k, kl, mid) > 0) a = mid + 1; else b = mid;
    }
    return a;
}

__global__ void __launch_bounds__(256) k_limit_decode(LimitParams p) {
    pdl_trigger();
    pdl_wait();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const uint4 r = p.rec[i];
    uint64_t kl = 0;
    const bool ok = limit_decode(r, &kl);
    uint32_t code = ok ? 0u : (r.z ? kScanStopPanic : kScanStopErr);
    const uint8_t *key = range_entry(r) + 8;
    p.flat[i] = make_uint4(r.x, r.y, (uint32_t)(8 + kl), r.w);
    p.pfx[i] = ok ? range_prefix(key, (uint32_t)kl) : 0ull;
    const uint32_t pr = p.rpair[i];
    const LimitPair pp = p.pairs[pr];
    const bool desc = p.queries[pp.query].desc;
    const uint32_t j = desc ? i + 1 : i - 1; // the neighbour: previous record (forward), next record (reverse)
    uint64_t nkl = 0;
    if (ok && (desc ? j < pp.first + pp.count : i > pp.first) && limit_decode(p.rec[j], &nkl)) {
        const int c = scan_key_cmp(range_entry(p.rec[j]) + 8, nkl, key, kl);
        if (desc ? c <= 0 : c >= 0) code = kLimitUnsorted;
    }
    p.code[i] = code;
    if (code) atomicMin(&p.pair_bad[pr], desc ? pp.first + pp.count - 1 - i : i - pp.first);
}

__global__ void __launch_bounds__(256) k_limit_query(LimitParams p) {
    pdl_trigger();
    pdl_wait();
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= p.n_queries) return;
    const LimitQuery Q = p.queries[q];
    const bool desc = Q.desc;
    for (uint32_t k = Q.pair0; k < Q.pair1; k++) {
        const uint32_t b = p.pair_bad[k];
        if (b != ~0u) {
            const LimitPair pp = p.pairs[k];
            p.qout[q] = make_uint4(0, p.code[desc ? pp.first + pp.count - 1 - b : pp.first + b], k, b);
            p.front[q] = ~0u;
            return;
        }
    }
    uint32_t best = ~0u;
    for (uint32_t k = Q.pair0; k < Q.pair1; k++) {
        const LimitPair pp = p.pairs[k];
        if (!pp.truncated || !pp.count) continue;
        const uint32_t j = desc ? pp.first : pp.first + pp.count - 1; // the staged record nearest the span's far end
        const uint4 r = p.flat[j];
        if (best == ~0u) { best = j; continue; }
        const int c = limit_cmp(p, j, p.pfx[j], range_entry(r) + 8, r.z - 8, best);
        if (desc ? c > 0 : c < 0) best = j;
    }
    for (uint32_t k = Q.pair0; k < Q.pair1; k++) {
        const LimitPair pp = p.pairs[k];
        bool set = false;
        if (best != ~0u && pp.truncated && pp.count) {
            const uint4 r = p.flat[best];
            set = limit_cmp(p, best, p.pfx[best], range_entry(r) + 8, r.z - 8, desc ? pp.first : pp.first + pp.count - 1) == 0;
        }
        p.setter[k] = set ? 1u : 0u;
    }
    p.front[q] = best;
    p.qout[q] = make_uint4(0, 0, ~0u, 0);
}

__global__ void __launch_bounds__(256) k_limit_flag(LimitParams p) {
    pdl_trigger();
    pdl_wait();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const uint32_t pr = p.rpair[i];
    const uint32_t q = p.pairs[pr].query;
    const LimitQuery Q = p.queries[q];
    bool keep = p.qout[q].y == 0;
    const uint4 r = p.flat[i];
    const uint8_t *k = range_entry(r) + 8;
    const uint32_t kl = r.z - 8;
    const unsigned long long pk = p.pfx[i];
    const uint32_t f = p.front[q];
    if (keep && f != ~0u) {
        const int c = limit_cmp(p, i, pk, k, kl, f);
        keep = Q.desc ? c >= 0 : c <= 0;
    }
    if (keep) keep = Q.keep_tombstones || ld_u64_unaligned_narrow(k + kl) != 0;
    for (uint32_t x = pr + 1; keep && x < Q.pair1; x++) { // a newer table staged the key
        const LimitPair pp = p.pairs[x];
        const uint32_t at = limit_lower_bound(p, pp, pk, k, kl);
        if (at < pp.first + pp.count && limit_cmp(p, i, pk, k, kl, at) == 0) keep = false;
    }
    p.keep[i] = keep ? 1u : 0u;
}

__global__ void __launch_bounds__(256) k_limit_rank(LimitParams p) {
    pdl_trigger();
    pdl_wait();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n_queries) {
        const LimitQuery Q = p.queries[i];
        p.qout[i].x = p.pre[Q.last] - p.pre[Q.first];
    }
    if (i >= p.n || p.pre[i + 1] == p.pre[i]) return;
    const uint32_t pr = p.rpair[i];
    const LimitPair mine = p.pairs[pr];
    const LimitQuery Q = p.queries[mine.query];
    const uint4 r = p.flat[i];
    const uint8_t *k = range_entry(r) + 8;
    const uint32_t kl = r.z - 8;
    const unsigned long long pk = p.pfx[i];
    // reverse: survivors after it in its pair, and every other pair's at or above its key (none there equals it)
    uint32_t rank = Q.desc ? p.pre[mine.first + mine.count] - p.pre[i + 1] : p.pre[i] - p.pre[mine.first];
    for (uint32_t x = Q.pair0; x < Q.pair1; x++) {
        if (x == pr) continue;
        const LimitPair pp = p.pairs[x];
        const uint32_t at = limit_lower_bound(p, pp, pk, k, kl);
        rank += Q.desc ? p.pre[pp.first + pp.count] - p.pre[at] : p.pre[at] - p.pre[pp.first];
    }
    p.rank[i] = rank;
}

__global__ void __launch_bounds__(256) k_limit_select(LimitParams p) {
    pdl_trigger();
    pdl_wait();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n || p.pre[i + 1] == p.pre[i]) return;
    const uint32_t q = p.pairs[p.rpair[i]].query, base = p.qsel[q], rank = p.rank[i];
    if (base == ~0u || rank >= p.queries[q].limit) return;
    p.sel_flat[base + rank] = p.flat[i];
    p.sel_dest[base + rank] = 0u;
}

} // namespace dbeel
