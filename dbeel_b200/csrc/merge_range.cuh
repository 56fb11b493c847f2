// merge_range.cuh -- the merge stage of dbeel_reader_get_range: one key-aligned partition of a reader's span records, split
// per destination by the scan chain (k_scan_classify .. k_route_scatter), becomes per destination the LAST version of every
// key, in ascending key order, tombstones dropped unless asked for.  It runs between k_route_scatter and
// k_scan_stream_carry and leaves what they leave -- a split (here: the compacted one, written over `flat`) and the totals
// counts | bytes | starts per destination -- so phase 2 (k_scan_tile_sums .. k_rebase_index) runs unchanged on it.
//
// After the split, destination d's segment holds its records in iteration order: one run per table, tables ascending, each
// run in record order.  On tables whose keys strictly ascend every run is sorted, so
//   superseded  = a later run of the segment holds the same key (one binary search per later run);
//   rank        = survivors before the record in its own run + survivors below its key in every other run (lower bound);
// and the survivors of a segment, scattered to segment start + rank, come out in key order with no sort.
//
//   k_range_keys      per split record: its table (the slice whose window holds the entry) and its big-endian 8-byte key
//                     prefix, so most comparisons of the searches are one 8-byte load
//   k_range_check     per partition record (flat, iteration order, every span record whatever its destination): its key is
//                     above its predecessor in the same table and inside the partition's key interval [lo, hi), else the
//                     error word is set (DBEEL_ERR_UNSORTED_RUN).  Checked in every partition, this is the strict ascent of
//                     every table's span records, since the partitions tile each table's spans in record order.
//   k_range_flag      per split record: keep = not superseded and (not a tombstone or tombstones kept)
//   k_range_tile_sums / k_range_tile_scan / k_range_prefix   exclusive prefix sum of keep over the split (pre[span] = all)
//   k_range_rank      per survivor: its merged position; the record goes to out[pre[segment start] + rank]
//   k_range_totals    one block: the new counts | bytes | starts, in the device totals and in the pinned header
//
// A partition with a stop (its stop word set, or an earlier partition's) is left as the split made it: rank copies the
// split through and the totals stay, so phase 2 reads only records before the stop.  The caller discards that output.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "device_fns.cuh"
#include "kernels.cuh"
#include "route.cuh"
#include "scan.cuh"

namespace dbeel {

constexpr int kRangeTile = 1024; // records per prefix-sum tile (one block)

struct RangeMergeParams {
    const ScanTable *tables;          // the partition's slices (ScanParams.tables)
    const uint32_t *slice_table;      // [n_slices] reader table of every slice
    uint32_t n_slices;
    uint32_t n;                       // partition records (flat)
    uint32_t n_ranges;
    uint32_t keep_tombstones;
    const uint4 *flat;                // [n] iteration order (k_scan_classify)
    const uint4 *split;               // [span] per destination (k_route_scatter)
    uint4 *out;                       // [span] the merged split (may alias flat: flat is read only by k_range_check)
    unsigned long long *totals;       // RouteParams.totals: counts | bytes | starts | stop word
    unsigned long long *pub;          // the partition's pinned header (k_route_starts' copy of the totals)
    uint32_t *tab;                    // [span] reader table per split record
    unsigned long long *pfx;          // [span] big-endian key prefix per split record
    uint32_t *pre;                    // [span + 1] keep, then its exclusive prefix sum
    uint32_t *tile;                   // [tiles + 1]
    unsigned long long *dbytes;       // [n_ranges] surviving bytes per destination (zero between partitions)
    uint32_t *err;                    // set by k_range_check: a table's span records do not strictly ascend
    const uint8_t *lo, *hi;           // the partition's key interval; null = open
    uint32_t lo_len, hi_len;
};

__device__ __forceinline__ bool range_stopped(const RangeMergeParams &p) { return p.totals[3 * p.n_ranges] != ~0ull; }

__device__ __forceinline__ uint32_t range_span(const RangeMergeParams &p) {
    const uint32_t nd = p.n_ranges;
    return (uint32_t)(p.totals[2 * nd + nd - 1] + p.totals[nd - 1]);
}

// entry address and key length of a split / flat record {source address, 8 + klen, full_size}
__device__ __forceinline__ const uint8_t *range_entry(const uint4 &r) {
    return reinterpret_cast<const uint8_t *>((uint64_t)r.x | ((uint64_t)r.y << 32));
}

__device__ __forceinline__ unsigned long long range_prefix(const uint8_t *key, uint32_t klen) {
    if (klen == 0) return 0ull;
    unsigned long long x = bswap64(ld_u64_unaligned_narrow(key));
    if (klen < 8) x &= ~0ull << (8 * (8 - klen));
    return x;
}

// Vec<u8>::cmp of split record j's key with (prefix, key, klen): the prefixes decide unless they tie
__device__ __forceinline__ int range_cmp_at(const RangeMergeParams &p, uint32_t j, unsigned long long pk, const uint8_t *k,
                                            uint32_t kl) {
    const unsigned long long pj = p.pfx[j];
    if (pj != pk) return pj < pk ? -1 : 1;
    const uint4 r = p.split[j];
    return scan_key_cmp(range_entry(r) + 8, r.z - 8, k, kl);
}

// first position in [a, b) of the split whose key is >= k (the run [a, b) ascending)
__device__ __forceinline__ uint32_t range_lower_bound(const RangeMergeParams &p, uint32_t a, uint32_t b, unsigned long long pk,
                                                      const uint8_t *k, uint32_t kl) {
    while (a < b) {
        const uint32_t mid = a + ((b - a) >> 1);
        if (range_cmp_at(p, mid, pk, k, kl) < 0) a = mid + 1; else b = mid;
    }
    return a;
}

// the end of the run that starts at j (records of table tab[j]) inside [j, e)
__device__ __forceinline__ uint32_t range_run_end(const RangeMergeParams &p, uint32_t j, uint32_t e) {
    const uint32_t t = p.tab[j];
    uint32_t a = j + 1, b = e;
    while (a < b) {
        const uint32_t mid = a + ((b - a) >> 1);
        if (p.tab[mid] == t) a = mid + 1; else b = mid;
    }
    return a;
}

// the first position of the run that holds i inside [s, i]
__device__ __forceinline__ uint32_t range_run_begin(const RangeMergeParams &p, uint32_t s, uint32_t i) {
    const uint32_t t = p.tab[i];
    uint32_t a = s, b = i;
    while (a < b) {
        const uint32_t mid = a + ((b - a) >> 1);
        if (p.tab[mid] < t) a = mid + 1; else b = mid;
    }
    return a;
}

// the destination segment [*s, *e) that holds split position i
__device__ __forceinline__ uint32_t range_segment(const unsigned long long *s_start, const unsigned long long *s_end, uint32_t nd,
                                                  uint32_t i, uint32_t *s, uint32_t *e) {
    uint32_t a = 0, b = nd; // first d whose end is > i
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (s_end[mid] <= i) a = mid + 1; else b = mid;
    }
    *s = (uint32_t)s_start[a];
    *e = (uint32_t)s_end[a];
    return a;
}

__global__ void __launch_bounds__(256) k_range_keys(RangeMergeParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ uintptr_t s_ix[kScanMaxTables];
    __shared__ uint32_t s_tab[kScanMaxTables];
    if (range_stopped(p)) return;
    for (uint32_t k = threadIdx.x; k < p.n_slices; k += blockDim.x) {
        s_ix[k] = reinterpret_cast<uintptr_t>(p.tables[k].index);
        s_tab[k] = p.slice_table[k];
    }
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= range_span(p)) return;
    const uint4 r = p.split[i];
    const uintptr_t a = reinterpret_cast<uintptr_t>(range_entry(r));
    uint32_t lo = 0, hi = p.n_slices; // the last slice whose index slice lies below the entry: its window holds it
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s_ix[mid] <= a) lo = mid; else hi = mid;
    }
    p.tab[i] = s_tab[lo];
    p.pfx[i] = range_prefix(range_entry(r) + 8, r.z - 8);
}

__global__ void __launch_bounds__(256) k_range_check(RangeMergeParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ uint32_t s_base[kScanMaxTables];
    __shared__ uint32_t s_tab[kScanMaxTables];
    if (range_stopped(p)) return;
    for (uint32_t k = threadIdx.x; k < p.n_slices; k += blockDim.x) {
        s_base[k] = p.tables[k].base;
        s_tab[k] = p.slice_table[k];
    }
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    auto table_of = [&](uint32_t x) {
        uint32_t lo = 0, hi = p.n_slices;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (s_base[mid] <= x) lo = mid; else hi = mid;
        }
        return s_tab[lo];
    };
    const uint4 r = p.flat[i];
    const uint8_t *k = range_entry(r) + 8;
    const uint32_t kl = r.z - 8;
    bool bad = (p.lo && scan_key_cmp(k, kl, p.lo, p.lo_len) < 0) || (p.hi && scan_key_cmp(k, kl, p.hi, p.hi_len) >= 0);
    if (!bad && i > 0 && table_of(i - 1) == table_of(i)) {
        const uint4 q = p.flat[i - 1];
        bad = scan_key_cmp(range_entry(q) + 8, q.z - 8, k, kl) >= 0;
    }
    if (bad) atomicOr(p.err, 1u);
}

__global__ void __launch_bounds__(256) k_range_flag(RangeMergeParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ unsigned long long s_start[kScanMaxRanges], s_end[kScanMaxRanges];
    if (range_stopped(p)) return;
    const uint32_t nd = p.n_ranges;
    for (uint32_t d = threadIdx.x; d < nd; d += blockDim.x) {
        s_start[d] = p.totals[2 * nd + d];
        s_end[d] = p.totals[2 * nd + d] + p.totals[d];
    }
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint32_t)s_end[nd - 1]) return;
    uint32_t s, e;
    range_segment(s_start, s_end, nd, i, &s, &e);
    const uint4 r = p.split[i];
    const uint8_t *ent = range_entry(r);
    const uint32_t kl = r.z - 8;
    bool keep = p.keep_tombstones || ld_u64_unaligned_narrow(ent + 8 + kl) != 0;
    const unsigned long long pk = p.pfx[i];
    for (uint32_t j = range_run_end(p, i, e); keep && j < e;) { // every later run of the segment
        const uint32_t je = range_run_end(p, j, e);
        const uint32_t at = range_lower_bound(p, j, je, pk, ent + 8, kl);
        if (at < je && range_cmp_at(p, at, pk, ent + 8, kl) == 0) keep = false;
        j = je;
    }
    p.pre[i] = keep ? 1u : 0u;
}

__global__ void __launch_bounds__(kRangeTile) k_range_tile_sums(RangeMergeParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ uint32_t s_w[kRangeTile / 32];
    if (range_stopped(p)) return;
    const uint32_t span = range_span(p);
    const uint32_t i = blockIdx.x * kRangeTile + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (blockIdx.x * kRangeTile >= span) return;
    uint32_t v = i < span ? p.pre[i] : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
    if (lane == 0) s_w[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < kRangeTile / 32; w++) t += s_w[w];
        p.tile[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kRangeTile) k_range_tile_scan(RangeMergeParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ unsigned long long s_b[32];
    __shared__ uint32_t s_c[32];
    if (range_stopped(p)) return;
    const uint32_t tiles = (range_span(p) + kRangeTile - 1) / kRangeTile;
    uint32_t carry = 0;
    for (uint32_t b0 = 0; b0 < tiles; b0 += kRangeTile) {
        const uint32_t b = b0 + threadIdx.x;
        unsigned long long vb = 0, tb;
        uint32_t vc = b < tiles ? p.tile[b] : 0u, tc;
        __syncthreads();
        block_excl_scan_1024(vb, vc, s_b, s_c, &tb, &tc);
        if (b < tiles) p.tile[b] = carry + vc;
        carry += tc;
    }
    if (threadIdx.x == 0) p.tile[tiles] = carry;
}

__global__ void __launch_bounds__(kRangeTile) k_range_prefix(RangeMergeParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ unsigned long long s_b[32];
    __shared__ uint32_t s_c[32];
    if (range_stopped(p)) return;
    const uint32_t span = range_span(p);
    if (blockIdx.x * kRangeTile >= span) return;
    const uint32_t i = blockIdx.x * kRangeTile + threadIdx.x;
    unsigned long long vb = 0, tb;
    uint32_t vc = i < span ? p.pre[i] : 0u, tc;
    block_excl_scan_1024(vb, vc, s_b, s_c, &tb, &tc);
    if (i < span) p.pre[i] = p.tile[blockIdx.x] + vc;
    if (i == 0) p.pre[span] = p.tile[(span + kRangeTile - 1) / kRangeTile];
}

__global__ void __launch_bounds__(256) k_range_rank(RangeMergeParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ unsigned long long s_start[kScanMaxRanges], s_end[kScanMaxRanges], s_bytes[kScanMaxRanges];
    const uint32_t nd = p.n_ranges;
    const bool stopped = range_stopped(p);
    for (uint32_t d = threadIdx.x; d < nd; d += blockDim.x) {
        s_start[d] = p.totals[2 * nd + d];
        s_end[d] = p.totals[2 * nd + d] + p.totals[d];
        s_bytes[d] = 0;
    }
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, span = (uint32_t)s_end[nd - 1];
    if (stopped || *p.err) {
        if (stopped && i < span) p.out[i] = p.split[i]; // left as the split made it
        return;
    }
    if (i < span && p.pre[i + 1] != p.pre[i]) {
        uint32_t s, e;
        const uint32_t d = range_segment(s_start, s_end, nd, i, &s, &e);
        const uint4 r = p.split[i];
        const uint8_t *k = range_entry(r) + 8;
        const uint32_t kl = r.z - 8;
        const unsigned long long pk = p.pfx[i];
        const uint32_t mine = range_run_begin(p, s, i);
        uint32_t rank = p.pre[i] - p.pre[mine];
        for (uint32_t j = s; j < e;) {
            const uint32_t je = range_run_end(p, j, e);
            if (j != mine) rank += p.pre[range_lower_bound(p, j, je, pk, k, kl)] - p.pre[j];
            j = je;
        }
        p.out[p.pre[s] + rank] = r;
        atomicAdd(&s_bytes[d], (unsigned long long)r.w);
    }
    __syncthreads();
    for (uint32_t d = threadIdx.x; d < nd; d += blockDim.x)
        if (s_bytes[d]) atomicAdd(&p.dbytes[d], s_bytes[d]);
}

__global__ void k_range_totals(RangeMergeParams p) {
    pdl_trigger();
    pdl_wait();
    const uint32_t nd = p.n_ranges;
    if (!range_stopped(p) && threadIdx.x == 0 && range_span(p)) { // an empty split keeps its zero totals
        const bool none = *p.err != 0;
        for (uint32_t d = 0; d < nd; d++) {
            const unsigned long long s = p.totals[2 * nd + d], e = s + p.totals[d];
            const unsigned long long a = p.pre[s], c = none ? 0ull : p.pre[e] - a, b = none ? 0ull : p.dbytes[d];
            p.totals[d] = p.pub[d] = c;
            p.totals[nd + d] = p.pub[nd + d] = b;
            p.totals[2 * nd + d] = p.pub[2 * nd + d] = a;
        }
    }
    __syncthreads();
    for (uint32_t d = threadIdx.x; d < nd; d += blockDim.x) p.dbytes[d] = 0;
    __threadfence_system();
}

} // namespace dbeel
