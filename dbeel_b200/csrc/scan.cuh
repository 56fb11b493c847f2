// scan.cuh -- LSMTree::iter_filter over a tree's SSTables on the GPU (src/storage_engine/lsm_tree.rs:133-282): every index
// record of every table, oldest table first, decoded like AsyncIter::read_one (:210-281) and sent to the first range that
// accepts it -- a murmur3_32 hash range compared with migration.rs's between_cmp (:54-60), or a key range [start, end).
//
//   k_scan_classify  one thread per index record: frame + timestamp checks, murmur3 / key compare, destination per record,
//                    atomicMin of the first record that stops the reference's iteration (and why)
//   k_scan_hist      per block: drop everything at or after the stop, count each destination (the input of k_route_scan)
//   k_route_scan / k_route_starts / k_route_scatter (route.cuh), unchanged: stable split into one stream per destination
//   k_scan_tile_sums per resolve tile: bytes of the split records (the input of k_scan_tiles / k_scan_chunks / k_emit)
//   k_emit, k_gather_h, k_rebase_index: the output .index, the payload copy, per-destination file offsets
//
// The records the split moves are 16 bytes {source address, 8 + key length, full_size}: the layout k_emit reads, so the
// payload is read once (k_gather_h) and nothing else touches it.
//
// Streamed (dbeel_scan_stream): one partition of the record sequence per chain, the tables' .data windows passed as biased
// pointers (ScanTable.data + offset = the entry inside the window), so k_scan_classify runs unchanged on partition-local
// positions.  k_scan_stream_carry sits between the split and phase 2 and replaces dbeel_scan's host round trip there.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "device_fns.cuh"
#include "kernels.cuh"
#include "route.cuh"

namespace dbeel {

constexpr uint32_t kScanMaxTables = 1024;   // = DBEEL_MAX_RUNS
constexpr uint32_t kScanMaxRanges = 256;    // = kRouteMaxShards: one split stream per destination
constexpr uint32_t kScanNone = 0xFFFFFFFFu; // destination of a record no range accepts (or at / past the stop)
// stop key = (global record position << 12) | (table << 2) | reason: the minimum is the first failing record in iteration
// order; an empty table fails at the position its first record would have had, ahead of the next table's record 0.
constexpr uint32_t kScanStopErr = 1u;   // next() returns Err: the entry does not deserialize
constexpr uint32_t kScanStopPanic = 2u; // the reference panics: full_size == 0, bytes past the end of .data, empty table

struct ScanTable {
    const uint8_t *data;
    uint64_t data_len;
    const uint4 *index;
    uint32_t n_rec; // floor(index_len / 16) (lsm_tree.rs:225, sizes from :453)
    uint32_t base;  // global position of the table's record 0
};

struct ScanParams {
    const ScanTable *tables;
    uint32_t n_tables;
    uint32_t n;        // records over all tables
    uint32_t key_kind; // 0: hash ranges, 1: key ranges
    uint32_t n_ranges;
    const uint32_t *hash_ranges;         // [2 n_ranges] (start, end)
    const uint8_t *keys;                 // key ranges: start_d = keys[off[2d] .. off[2d+1]), end_d = keys[off[2d+1] .. off[2d+2])
    const unsigned long long *key_off;   // [2 n_ranges + 1]
    uint32_t *dest;                      // [n] destination per record
    uint4 *flat;                         // [n] {source address, 8 + klen, full_size} per record
    unsigned long long *stop;            // first failing record (key above), ~0 = none
    unsigned long long stop0;            // the host's stop key for the first empty table, ~0 = none
};

// migration.rs:54-60, literally: for end < start it accepts every hash, for start == end none.
DB_HD bool scan_between_cmp(uint32_t hash, uint32_t start, uint32_t end) {
    if (end < start) return hash < start || hash >= end;
    return hash >= start && hash < end;
}

// Vec<u8>::cmp of two byte strings in global memory, 8 bytes per step.  Loads may read up to 7 bytes past either string.
__device__ __forceinline__ int scan_key_cmp(const uint8_t *a, uint64_t al, const uint8_t *b, uint64_t bl) {
    const uint64_t m = al < bl ? al : bl;
    for (uint64_t q = 0; q < m; q += 8) {
        uint64_t x = bswap64(ld_u64_unaligned_narrow(a + q)), y = bswap64(ld_u64_unaligned(b + q));
        if (m - q < 8) {
            const uint32_t drop = (uint32_t)(8 - (m - q)) * 8;
            x >>= drop;
            y >>= drop;
        }
        if (x != y) return x < y ? -1 : 1;
    }
    return al < bl ? -1 : (al > bl ? 1 : 0);
}

__global__ void __launch_bounds__(256) k_scan_classify(ScanParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ uint32_t s_base[kScanMaxTables];
    __shared__ uint32_t s_hash[2 * kScanMaxRanges];
    __shared__ unsigned long long s_koff[2 * kScanMaxRanges + 1];
    for (uint32_t t = threadIdx.x; t < p.n_tables; t += blockDim.x) s_base[t] = p.tables[t].base;
    if (p.key_kind) {
        for (uint32_t k = threadIdx.x; k <= 2 * p.n_ranges; k += blockDim.x) s_koff[k] = p.key_off[k];
    } else {
        for (uint32_t k = threadIdx.x; k < 2 * p.n_ranges; k += blockDim.x) s_hash[k] = p.hash_ranges[k];
    }
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    uint32_t lo = 0, hi = p.n_tables; // last table whose base is <= i: an empty table shares its successor's base
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s_base[mid] <= i) lo = mid; else hi = mid;
    }
    const ScanTable &t = p.tables[lo];
    const uint4 rec = __ldg(&t.index[i - s_base[lo]]); // EntryOffset: offset u64, key_size u32 (ignored), full_size u32
    const uint64_t off = (uint64_t)rec.x | ((uint64_t)rec.y << 32);
    const uint64_t fs = rec.w;
    uint32_t reason = 0, d = kScanNone;
    uint64_t klen = 0;
    if (fs == 0 || off > t.data_len || fs > t.data_len - off) {
        reason = kScanStopPanic; // read_at's assert_ne!(size, 0) / the slice past the file's end (cached_file_reader.rs:68,82)
    } else {
        // bincode Entry from exactly fs bytes: u64 klen | key | u64 dlen | data | i128 ts, no trailing bytes
        const uint8_t *e = t.data + off;
        bool ok = fs >= 8;
        if (ok) {
            klen = ld_u64_unaligned_narrow(e);
            ok = klen <= fs - 8 && fs - 8 - klen >= 8;
        }
        if (ok) {
            const uint64_t dlen = ld_u64_unaligned_narrow(e + 8 + klen);
            const uint64_t rest = fs - 16 - klen;
            ok = dlen <= rest && rest - dlen == 16 &&
                 ts_decodes(ld_u64_unaligned_narrow(e + fs - 16), ld_u64_unaligned_narrow(e + fs - 8));
        }
        if (!ok) {
            reason = kScanStopErr;
        } else if (p.key_kind == 0) {
            const uint8_t *key = e + 8;
            const uint32_t h = murmur3_32(klen, 0u, [key](uint64_t q) { return ld_u64_unaligned_narrow(key + 8 * q); });
            for (uint32_t r = 0; r < p.n_ranges; r++)
                if (scan_between_cmp(h, s_hash[2 * r], s_hash[2 * r + 1])) { d = r; break; }
        } else {
            const uint8_t *key = e + 8;
            for (uint32_t r = 0; r < p.n_ranges; r++) {
                const uint64_t s0 = s_koff[2 * r], s1 = s_koff[2 * r + 1], s2 = s_koff[2 * r + 2];
                if (scan_key_cmp(p.keys + s0, s1 - s0, key, klen) <= 0 && scan_key_cmp(key, klen, p.keys + s1, s2 - s1) < 0) {
                    d = r;
                    break;
                }
            }
        }
    }
    if (reason) atomicMin(p.stop, ((unsigned long long)i << 12) | ((unsigned long long)lo << 2) | reason);
    const unsigned long long src = reinterpret_cast<unsigned long long>(t.data + off);
    p.flat[i] = make_uint4((uint32_t)src, (uint32_t)(src >> 32), (uint32_t)(8 + klen), (uint32_t)fs);
    p.dest[i] = d;
}

// One block per kRouteThreads records, the blocks of k_route_scan / k_route_scatter: records at or past the stop are
// dropped (the reference never delivers them), the rest are counted per destination; payload bytes per destination.
__global__ void __launch_bounds__(kRouteThreads) k_scan_hist(ScanParams sp, RouteParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ uint32_t s_cnt[kScanMaxRanges];
    __shared__ unsigned long long s_bytes[kScanMaxRanges];
    const uint32_t tid = threadIdx.x;
    for (uint32_t s = tid; s < p.n_shards; s += kRouteThreads) { s_cnt[s] = 0; s_bytes[s] = 0; }
    __syncthreads();
    const unsigned long long stop = *sp.stop < sp.stop0 ? *sp.stop : sp.stop0;
    const unsigned long long stop_pos = stop >> 12;
    const uint32_t i = blockIdx.x * (uint32_t)kRouteThreads + tid;
    if (i < p.n) {
        uint32_t d = p.shard_of[i];
        if ((unsigned long long)i >= stop_pos && d != kScanNone) {
            d = kScanNone;
            p.shard_of[i] = d;
        }
        if (d != kScanNone) {
            atomicAdd(&s_cnt[d], 1u);
            atomicAdd(&s_bytes[d], (unsigned long long)p.index[i].w);
        }
    }
    __syncthreads();
    for (uint32_t s = tid; s < p.n_shards; s += kRouteThreads) {
        p.hist[(uint64_t)blockIdx.x * p.n_shards + s] = s_cnt[s];
        if (s_bytes[s]) atomicAdd(&p.totals[p.n_shards + s], s_bytes[s]);
    }
}

// Per resolve tile (kResolveThreads split records): bytes and entries, the aggregates k_scan_tiles scans.  The split's
// length is Ctl.span, so the grid may be sized from a bound (streamed partitions).
__global__ void __launch_bounds__(kResolveThreads) k_scan_tile_sums(Params p, const uint4 *split) {
    pdl_trigger();
    pdl_wait();
    __shared__ unsigned long long s_b[kResolveThreads / 32];
    const uint32_t span = p.ctl->span;
    if (blockIdx.x * (uint32_t)kResolveThreads >= span) return;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t i = blockIdx.x * (uint32_t)kResolveThreads + tid;
    unsigned long long b = i < span ? (unsigned long long)split[i].w : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) b += __shfl_down_sync(0xFFFFFFFFu, b, o);
    if (lane == 0) s_b[warp] = b;
    __syncthreads();
    if (tid == 0) {
        unsigned long long tb = 0;
        for (int w = 0; w < kResolveThreads / 32; w++) tb += s_b[w];
        const uint32_t i0 = blockIdx.x * (uint32_t)kResolveThreads;
        p.tile_bytes[blockIdx.x] = tb;
        p.tile_count[blockIdx.x] = span - i0 < (uint32_t)kResolveThreads ? span - i0 : (uint32_t)kResolveThreads;
    }
}

// Streamed scans: one thread, after k_route_starts of a partition (totals = counts | bytes | starts | stop, nd each + 1).
// carry[2 nd + 1] (device, zeroed before the first partition) = .data bytes | entries every destination received from the
// partitions before, | halted (an earlier partition found the stop).  Partitions run in order on one stream, so this is
// exact with no host in the loop.  The thread
//   * publishes the carry before this partition behind k_route_starts's totals in the mapped pinned header (pub[3 nd + 1 ..
//     5 nd + 1] and the halted word at pub[5 nd + 1]): the host learns the exact D2H sizes and the file offsets from it;
//   * makes k_rebase_index write destination-file offsets across partitions: mem_table[2d] = (bytes before d in this
//     partition) - carry bytes of d, so off - mem_table[2d] = offset inside d's part here + what d had before (mod 2^64);
//   * sets Ctl.span / total for phase 2, whose grids come from the host's bound;
//   * adds the partition to the carry, and arms the next partition's stop word: 0 once halted (k_scan_hist then drops every
//     record: nothing is delivered after the reference's iteration ended), else none.
__global__ void k_scan_stream_carry(RouteParams rp, Params p, unsigned long long *carry, unsigned long long *pub) {
    pdl_trigger();
    pdl_wait();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const uint32_t nd = rp.n_shards;
    unsigned long long *tot = rp.totals;
    const unsigned long long halted = carry[2 * nd];
    unsigned long long before = 0, items = 0;
    for (uint32_t d = 0; d < nd; d++) {
        const unsigned long long cb = carry[d], ci = carry[nd + d], b = tot[nd + d], n = tot[d];
        pub[3 * nd + 1 + d] = cb;
        pub[4 * nd + 1 + d] = ci;
        p.mem_table[2 * d] = before - cb;
        p.mem_table[2 * d + 1] = tot[2 * nd + d];
        carry[d] = cb + b;
        carry[nd + d] = ci + n;
        before += b;
        items += n;
    }
    p.mem_table[2 * nd] = before;
    p.mem_table[2 * nd + 1] = items;
    pub[5 * nd + 1] = halted;
    Ctl *c = p.ctl;
    c->flags = 0;
    c->span = c->total = (uint32_t)items;
    c->out_data_len = 0;
    c->out_items = 0;
    const bool halts = halted || tot[3 * nd] != ~0ull;
    carry[2 * nd] = halts ? 1ull : 0ull;
    tot[3 * nd] = halts ? 0ull : ~0ull;
    __threadfence_system();
}

} // namespace dbeel
