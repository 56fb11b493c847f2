// kernels.cuh -- sm_90a kernels of the compaction engine.  See DESIGN.md for the pipeline.
//
// All work on this path is byte / integer work bounded by HBM bandwidth; there is no dense
// contraction, so no tensor-core code.  What matters: 128-bit coalesced loads and stores,
// moving only 16-byte merge records (never payload) through the merge passes, and touching
// every payload byte exactly once (one read, one write) in the gather kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "device_fns.cuh"

namespace dbeel {

// ------------------------------------------------------------------------------------
// device-side job description

struct RunDesc {
    const uint8_t *data; // address of .data byte 0 (biased by -off_base when only a slice of the file is resident)
    uint64_t data_len;   // .data offsets below this bound are resident
    uint64_t off_base;   // ... and at or above this one; the first record of the (slice of the) run starts here
    const uint4 *index;
    uint32_t n_in; // index records of the (slice of the) run
    uint32_t base; // gid of this run's first entry
};

struct Seg {
    uint32_t start, len;
};

enum : uint32_t {
    kFlagTruncated = 1u,   // some run ended before its last index record
    kFlagUnsorted = 2u,    // a valid entry does not carry the job's common key prefix
    kFlagVerifyFailed = 4u, // DBEEL_FLAG_VERIFY_SORTED found a descent or duplicate
    // DBEEL_FLAG_REFERENCE_READER only (lsm_tree.rs:1158-1170 never looks at `offset` / `key_size`):
    kFlagIndexDiffers = 8u, // some index record disagrees with what a sequential read of .data yields
    kFlagRepaired = 16u     // ... so the job runs on a canonical copy of the index (k_ref_repair)
};

struct Ctl {
    uint32_t prefix_len;
    uint32_t flags;
    uint32_t total;  // entries that take part in the merge (sum of valid counts)
    uint32_t span;   // merged positions to walk: == total, except flush-many where every memtable keeps its gid range
    unsigned long long out_data_len;
    uint32_t out_items;
    uint32_t runs_truncated;
    uint8_t prefix[256];
};

constexpr int kMergeThreads = 256;
#ifndef DBEEL_MERGE_VT
#define DBEEL_MERGE_VT 7
#endif
#ifndef DBEEL_MERGE_CTAS
#define DBEEL_MERGE_CTAS 3
#endif
constexpr int kMergeVT = DBEEL_MERGE_VT; // odd: threads walk smem at a 112-byte stride -> no bank conflicts
constexpr int kMergeCtasPerSM = DBEEL_MERGE_CTAS; // persistent merge CTAs per SM
constexpr int kMergeTile = kMergeThreads * kMergeVT; // 1792 records = 28 KB of smem
#ifndef DBEEL_RESOLVE_THREADS
#define DBEEL_RESOLVE_THREADS 128
#endif
constexpr int kResolveThreads = DBEEL_RESOLVE_THREADS;
#ifndef DBEEL_GATHER_THREADS
#define DBEEL_GATHER_THREADS 128
#endif
constexpr int kGatherThreads = DBEEL_GATHER_THREADS; // 128 threads = 8 KB tiles at 12 CTAs/SM
constexpr int kGatherVecsPerThread = 4;

constexpr unsigned long long kGatherTileBytes = 16ull * kGatherThreads * kGatherVecsPerThread; // 16 KB of output per CTA
constexpr int kGatherMaxEntries = (int)(kGatherTileBytes / 32) + 2; // entries are >= 32 bytes
constexpr int kMaxLevels = 16;      // >= ceil(log2(DBEEL_MAX_RUNS)); flush: 2^16 sort tiles of kMergeTile (1792) arrivals

struct BloomParams {
    uint32_t *words;     // bit-vec storage inside the .bloom buffer (file offset 8); null = off
    uint64_t bits;       // bitmap_bits
    uint64_t bits_magic; // floor(2^64 / bits)
    uint32_t k_num;
    uint64_t sip[4]; // k0,k1 of hasher 0 ; k0,k1 of hasher 1
};

// Several independent jobs in one launch sequence.  A *group* is one of them: a memtable of dbeel_flush_many (one run) or
// a compaction of dbeel_compact_many (a block of consecutive runs).  Every group owns an aligned block of leaf
// segments, so merges never pair segments of two groups, and after the last level seg[n_levels][g] IS group g's
// merged slice.
struct GroupDesc {
    uint32_t first_run, n_runs; // compact-many: the job's runs
    uint32_t pos_end;           // compact-many: one past the job's last record position (start of its padding segments)
    int keep_tombstones;
    BloomParams bloom;          // compact-many: the job's own filter (words == null: none)
};

struct Params {
    const RunDesc *runs;
    uint32_t n_runs;
    uint32_t n_total; // sum of n_in
    uint32_t *first_bad;      // [n_runs] in: n_in, out: valid entry count
    uint32_t *first_mismatch; // [n_runs] first entry lacking the common prefix
    Ctl *ctl;
    Seg *seg[kMaxLevels + 1];       // seg[l][j]: sorted segment j entering level l
    uint32_t *tile_base[kMaxLevels]; // [pairs_l + 1] exclusive tile counts per pair
    uint32_t nseg[kMaxLevels + 1];
    uint32_t n_levels;
    uint32_t *part; // merge-path split points of the current level
    uint4 *bnd;          // [boundaries of the current level] {first A record, first B record, first output record} after the boundary (absolute)
    uint32_t *tile_bnd;  // [tiles of the current level] index of the boundary a tile starts at (its end is the next one)
    Rec *rec_a, *rec_b;
    // resolve / scan
    unsigned long long *tile_bytes; // [resolve tiles] bytes emitted by the tile, then (k_scan_tiles) bytes before it
    uint32_t *tile_count;           // [resolve tiles] same for entries
    unsigned long long *chunk_bytes; // [resolve tiles / 1024] the same one level up
    uint32_t *chunk_count;
    int keep_tombstones;
    int mode_flush; // 1: arrival batch -- winner = last arrival, tombstones kept
    uint32_t flush_slots;   // flush-many: leaf segments (sort tiles) reserved per memtable, a power of two; 0 otherwise
    uint32_t flush_ref_run; // flush: the batch whose first arrival seeds the common-prefix reduction
    uint32_t sparse_offsets; // WAL replay: index offsets point into the log, records do not abut (no running-offset check)
    uint32_t ref_reader;     // DBEEL_FLAG_REFERENCE_READER: decode runs exactly like read_next_entry (lsm_tree.rs:1158-1170)
    uint4 *fix_index;        // [n_total] canonical index records, written only when an input index disagrees with its .data
    uint32_t n_groups;         // flush-many: memtables, compact-many: jobs, 0 for a single job
    uint32_t group_slots;      // compact-many: leaf segments reserved per job (runs padded to a power of two), else 0
    const GroupDesc *groups;   // compact-many only
    unsigned long long *mem_table; // [n_groups + 1][2] = {.data bytes, entries} emitted before each group
    // outputs
    uint8_t *out_data;
    uint4 *out_index;
    unsigned long long *src_ptr; // [n_total] device address of each surviving entry's bytes
    uint32_t *tile_first;        // [ceil(data bytes / 16 KB) + 2] entry holding each gather tile's first byte
    uint32_t tile_first_n;       // gather tiles the buffers were sized for (sparse batches: the caller's bound may be too low)
    unsigned long long data_bound; // .data bytes the job checked against out->data_cap: k_gather_h writes nothing at or past it
    unsigned long long out_offset_base; // .data bytes written by earlier key-range partitions of the same output file
    BloomParams bloom;
    uint4 *hash_rec; // [n_total] {h0, h1} = both SipHash-1-3 values of every entry's key (k_extract), or null: the gather hashes
    uint32_t bloom_ctas;      // k_gather32<.., kSplit>: filter blocks interleaved with the copy blocks of the grid
    uint32_t bloom_elsewhere; // 1: k_bloom_res fills the filter on a second stream, next to the gather (which then skips it)
    // fused resolve + emit (single jobs): chained scan of the tiles' (bytes, entries), decoupled look-back
    uint32_t fin_tile;   // k_merge_final: nominal records per tile of the LAST level (< kMergeTile: room for the extensions), 0 = off
    uint32_t *part_ext;  // [boundaries of the last level] records with the boundary's key that follow it in A (bits 0-7) and B (8-15)
    unsigned long long *scan_state; // [resolve tiles][2]: {status << 62 | bytes, status << 32 | entries}, zeroed per job
    uint32_t *scan_ticket;          // tiles are numbered in the order their CTAs start
};

// ------------------------------------------------------------------------------------
// Programmatic dependent launch (sm_90+).  Every kernel of a job starts with trigger + wait: the trigger lets the NEXT kernel
// of the stream be scheduled while this one drains (its CTAs become resident as slots free up, launch latency and prologue
// hidden), the wait blocks until every earlier kernel has completed and flushed -- so ordering and visibility are exactly
// those of plain stream order.  Both are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ------------------------------------------------------------------------------------
// small load helpers

// Loads for RANDOM accesses (entry headers, index records reached through a gid, timestamps): the
// default L2 policy pulls a whole 128-byte line from HBM on a miss, four times what a 32-byte
// header needs.  The .L2::64B qualifier caps the fetch at the 64-byte HBM access granule.
__device__ __forceinline__ uint64_t ldg64_narrow(const uint64_t *q) {
    uint64_t v;
    asm volatile("ld.global.nc.L2::64B.u64 %0, [%1];" : "=l"(v) : "l"(q));
    return v;
}
__device__ __forceinline__ uint4 ldg128_narrow(const uint4 *q) {
    uint4 v;
    asm volatile("ld.global.nc.L2::64B.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(q));
    return v;
}
__device__ __forceinline__ uint64_t ld_u64_unaligned_narrow(const uint8_t *p) {
    uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint64_t *q = reinterpret_cast<const uint64_t *>(a & ~uintptr_t(7));
    uint32_t sh = (uint32_t)(a & 7) * 8;
    uint64_t lo = ldg64_narrow(q);
    if (sh == 0) return lo;
    uint64_t hi = ldg64_narrow(q + 1);
    return (lo >> sh) | (hi << (64 - sh));
}

__device__ __forceinline__ uint64_t ld_u64_unaligned(const uint8_t *p) {
    // two aligned 8-byte loads; the second is only issued when it holds needed bytes
    uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint64_t *q = reinterpret_cast<const uint64_t *>(a & ~uintptr_t(7));
    uint32_t sh = (uint32_t)(a & 7) * 8;
    uint64_t lo = __ldg(q);
    if (sh == 0) return lo;
    uint64_t hi = __ldg(q + 1);
    return (lo >> sh) | (hi << (64 - sh));
}

// Per-instruction L2 cache policy (it travels in the access's memory descriptor; no device-level carve-out).  The gather
// streams ~4 GB of payload through the 50 MB L2 while the bloom filter (~10 MB at the benchmark shapes) takes scattered
// REDs: marking the REDs evict_last keeps filter sectors resident between two touches.
__device__ __forceinline__ uint64_t l2_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void red_or_keep(uint32_t *q, uint32_t v, uint64_t pol) {
    asm volatile("red.global.or.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(q), "r"(v), "l"(pol) : "memory");
}

__device__ __forceinline__ Rec ld_rec(const Rec *p) {
    uint4 v = *reinterpret_cast<const uint4 *>(p);
    Rec r;
    r.x = v.x; r.y = v.y; r.z = v.z; r.w = v.w;
    return r;
}
__device__ __forceinline__ void st_rec(Rec *p, const Rec &r) {
    *reinterpret_cast<uint4 *>(p) = make_uint4(r.x, r.y, r.z, r.w);
}

// run that owns gid: the last run whose base <= gid (empty runs share a base with their
// successor, and the successor is the owner)
__device__ __forceinline__ uint32_t find_run(const Params &p, uint32_t gid) {
    uint32_t lo = 0, hi = p.n_runs; // answer in [lo, hi)
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (p.runs[mid].base <= gid) lo = mid; else hi = mid;
    }
    return lo;
}

// the group whose merged slice holds position i: last g with seg[n_levels][g].start <= i (empty groups share a start)
__device__ __forceinline__ uint32_t find_group(const Params &p, uint32_t i) {
    const Seg *fin = p.seg[p.n_levels];
    uint32_t lo = 0, hi = p.n_groups;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (fin[mid].start <= i) lo = mid; else hi = mid;
    }
    return lo;
}

struct KeyRef {
    const uint8_t *ptr; // first key byte
    uint32_t klen;
    const uint8_t *entry;
    uint32_t full_size;
};

__device__ __forceinline__ KeyRef key_of_gid(const Params &p, uint32_t gid) {
    uint32_t r = find_run(p, gid);
    const RunDesc &rd = p.runs[r];
    uint4 rec = __ldg(&rd.index[gid - rd.base]);
    uint64_t off = (uint64_t)rec.x | ((uint64_t)rec.y << 32);
    KeyRef k;
    k.entry = rd.data + off;
    k.ptr = k.entry + 8;
    k.klen = rec.z - 8;
    k.full_size = rec.w;
    return k;
}

// Vec<u8>::cmp of two keys known to agree on their first `skip` bytes (slow path).
__device__ __noinline__ int full_key_cmp(const Params &p, uint32_t ga, uint32_t gb, uint32_t skip) {
    KeyRef a = key_of_gid(p, ga), b = key_of_gid(p, gb);
    uint32_t m = a.klen < b.klen ? a.klen : b.klen;
    for (uint32_t i = skip; i < m; i++) {
        uint8_t ca = __ldg(a.ptr + i), cb = __ldg(b.ptr + i);
        if (ca != cb) return ca < cb ? -1 : 1;
    }
    return a.klen < b.klen ? -1 : (a.klen > b.klen ? 1 : 0);
}

// strict key order: a < b  (mod.rs:77-79; ties are left to the caller = stable merge)
__device__ __forceinline__ bool key_less(const Params &p, uint32_t skip, const Rec &a, const Rec &b) {
    int und;
    int c = rec_cmp_window(a, b, &und);
    if (und) c = full_key_cmp(p, a.w, b.w, skip);
    return c < 0;
}

// a < b for two records that sit in shared memory, touching as few bytes as decide the order: the
// first 8 key bytes (one LDS.64 each) settle almost every probe of a merge-path search; the third
// word and the gid are only read on a tie.  The searches are the main consumers of shared-memory
// bandwidth in the merge kernels, so this halves their traffic.
__device__ __forceinline__ bool key_less_smem(const Params &p, uint32_t skip, const Rec *a, const Rec *b) {
    const uint2 ax = *reinterpret_cast<const uint2 *>(a), bx = *reinterpret_cast<const uint2 *>(b);
    if (ax.x != bx.x) return ax.x < bx.x;
    if (ax.y != bx.y) return ax.y < bx.y;
    const uint2 az = *reinterpret_cast<const uint2 *>(&a->z), bz = *reinterpret_cast<const uint2 *>(&b->z);
    if (az.x != bz.x) return az.x < bz.x;
    if ((az.x & 0xFF) == kClampBeyond) return full_key_cmp(p, az.y, bz.y, skip) < 0;
    return false;
}

__device__ __forceinline__ bool key_equal(const Params &p, uint32_t skip, const Rec &a, const Rec &b) {
    int und;
    int c = rec_cmp_window(a, b, &und);
    if (und) c = full_key_cmp(p, a.w, b.w, skip);
    return c == 0;
}

// ------------------------------------------------------------------------------------
// K0: common key prefix of the job (one warp).
//
// Keys ascend inside a run, so the prefix shared by a run's first and last key is shared by
// every key in between; the job's prefix is the prefix common to all first/last keys.
// mode 0: speculative, uses n_in (index records are bounds-checked, nothing else);
// mode 1: runs only if some run was truncated, uses the validated counts;
// mode 2: runs only after an index repair (reference reader), speculative again on the canonical index.
// mode_flush: arrival batches are not sorted -> no prefix is skipped (L = 0).

__device__ __forceinline__ bool safe_key(const RunDesc &rd, uint32_t i, const uint8_t **ptr, uint32_t *klen) {
    uint4 rec = __ldg(&rd.index[i]);
    uint64_t off = (uint64_t)rec.x | ((uint64_t)rec.y << 32);
    if (rec.z < 8 || off < rd.off_base || off > rd.data_len || (uint64_t)rec.z > rd.data_len - off) return false;
    *ptr = rd.data + off + 8;
    *klen = rec.z - 8;
    return true;
}

__global__ void k_common_prefix(Params p, int mode) {
    pdl_trigger();
    pdl_wait();
    Ctl *c = p.ctl;
    if (mode == 1 && !(c->flags & kFlagTruncated)) return;
    if (mode == 2 && !(c->flags & kFlagRepaired)) return;
    const int validated = mode == 1;
    const uint32_t lane = threadIdx.x;
    __shared__ const uint8_t *s_ref;
    __shared__ uint32_t s_ref_len;
    if (lane == 0) { s_ref = nullptr; s_ref_len = 0; }
    __syncwarp();
    if (validated)
        for (uint32_t r = lane; r < p.n_runs; r += 32) p.first_mismatch[r] = 0xFFFFFFFFu;
    // reference key: first key of the first non-empty run
    if (lane == 0 && !p.mode_flush) {
        for (uint32_t r = 0; r < p.n_runs; r++) {
            uint32_t cnt = validated ? p.first_bad[r] : p.runs[r].n_in;
            if (!cnt) continue;
            const uint8_t *ptr; uint32_t kl;
            if (safe_key(p.runs[r], 0, &ptr, &kl)) { s_ref = ptr; s_ref_len = kl; }
            break; // an unreadable first record means L = 0 (safe)
        }
    }
    __syncwarp();
    const uint8_t *ref = s_ref;
    uint32_t L = s_ref_len < kMaxPrefix ? s_ref_len : kMaxPrefix;
    if (ref == nullptr) L = 0;
    // one lane per (run, first | last key): 16 keys of an 8-way job are compared at once, eight bytes per step
    for (uint32_t q = lane; q < 2 * p.n_runs && L; q += 32) {
        const uint32_t r = q >> 1, which = q & 1;
        uint32_t cnt = validated ? p.first_bad[r] : p.runs[r].n_in;
        if (!cnt) continue;
        const uint8_t *ptr; uint32_t kl;
        if (!safe_key(p.runs[r], which ? cnt - 1 : 0, &ptr, &kl)) { L = 0; break; }
        const uint32_t m = kl < L ? kl : L;
        uint32_t i = 0;
        bool diff = false;
        while (i + 8 <= m) { // aligned 8-byte words that hold a needed byte lie inside the mapped buffers
            const uint64_t x = ld_u64_unaligned(ptr + i) ^ ld_u64_unaligned(ref + i);
            if (x) { i += (uint32_t)(__ffsll((long long)x) - 1) >> 3; diff = true; break; }
            i += 8;
        }
        if (!diff) while (i < m && __ldg(ptr + i) == __ldg(ref + i)) i++;
        L = i;
    }
    for (int o = 16; o; o >>= 1) {
        uint32_t other = __shfl_xor_sync(0xFFFFFFFFu, L, o);
        L = other < L ? other : L;
    }
    for (uint32_t i = lane; i < L; i += 32) c->prefix[i] = __ldg(ref + i);
    if (lane == 0) c->prefix_len = L;
}

// ------------------------------------------------------------------------------------
// K1: validate every index record + entry header and extract the 16-byte merge record.
//
// "Valid" restates what the reference's sequential reader needs to decode entry i
// (lsm_tree.rs:1158-1170): the record lies inside .data at the running offset and
// bincode-decodes with no trailing bytes (klen/dlen prefixes agree with key_size/full_size).
// The first invalid entry ends its run (lsm_tree.rs:1014,1063): first_bad[r] = min index.

#ifndef DBEEL_EXTRACT_EPT
#define DBEEL_EXTRACT_EPT 2
#endif
#ifndef DBEEL_EXTRACT_MINB
#define DBEEL_EXTRACT_MINB 4
#endif
constexpr int kExtractEPT = DBEEL_EXTRACT_EPT; // entries per thread = independent load chains in flight per thread

// kRef = DBEEL_FLAG_REFERENCE_READER.  read_next_entry (lsm_tree.rs:1158-1170) consults `full_size` only: the record's
// bytes are the next full_size bytes of the .data stream (whatever `offset` says), the key length is the one bincode
// finds in those bytes (whatever `key_size` says), and an i128 outside `time`'s range fails the decode
// (utils/timestamp_nanos.rs:15-24).  The default mode instead treats a wrong offset / key_size as an undecodable record.
// With kRef the first pass only NOTES a disagreement (kFlagIndexDiffers); k_ref_repair then rebuilds a canonical index
// (offset = running sum of full_size, key_size = 8 + the length prefix found in .data) and pass `mode 2` validates that.
// mode 0: full validation; mode 1: only if a run was truncated -- re-extract with the shorter prefix; mode 2: full
// validation again, only after a repair.
// kPersist: launched with a grid that fits the GPU once (DBEEL_EXTRACT_PERSIST CTAs per SM); every thread walks several steps
// and fetches the NEXT step's index records before it starts on the current step's entry headers, so a step exposes one DRAM
// round trip (the headers) instead of two (index record, then header).
#ifndef DBEEL_EXTRACT_PERSIST_MINB
#define DBEEL_EXTRACT_PERSIST_MINB 3
#endif
template <bool kNarrow, bool kRef, bool kHash, bool kPersist = false>
__global__ void __launch_bounds__(256, kRef ? 3 : (kPersist ? DBEEL_EXTRACT_PERSIST_MINB : DBEEL_EXTRACT_MINB)) k_extract(Params p, int mode) {
    pdl_trigger();
    pdl_wait();
    auto ldu = [](const uint8_t *q) { return kNarrow ? ld_u64_unaligned_narrow(q) : ld_u64_unaligned(q); };
    Ctl *c = p.ctl;
    if (mode == 1 && !(c->flags & kFlagTruncated)) return;
    if (mode == 2 && !(c->flags & kFlagRepaired)) return;
    const bool redo = mode == 1;
    const uint32_t L = c->prefix_len;
    const uint64_t *pfx = reinterpret_cast<const uint64_t *>(c->prefix); // 8-byte aligned inside Ctl
    const uint32_t npw = (L + 7) >> 3;
    constexpr uint32_t STEP = 256u * kExtractEPT;
    // index records of a step (and their predecessors', for the running-offset check), fetched a step ahead when kPersist
    uint4 n_rec[kExtractEPT], n_pr[kExtractEPT];
    uint32_t n_run[kExtractEPT];
    auto fetch = [&](uint64_t g0n, uint4 rec[kExtractEPT], uint4 pr[kExtractEPT], uint32_t run[kExtractEPT]) {
#pragma unroll
        for (int u = 0; u < kExtractEPT; u++) {
            const uint64_t gg = g0n + u * 256u;
            rec[u] = pr[u] = make_uint4(0, 0, 0, 0);
            run[u] = 0;
            if (gg >= p.n_total) continue;
            run[u] = find_run(p, (uint32_t)gg);
            const RunDesc &rd = p.runs[run[u]];
            const uint32_t ii = (uint32_t)gg - rd.base;
            rec[u] = __ldg(&rd.index[ii]);
            if (ii && !redo) pr[u] = __ldg(&rd.index[ii - 1]);
        }
    };
    if (kPersist) fetch((uint64_t)blockIdx.x * STEP + threadIdx.x, n_rec, n_pr, n_run);
    for (uint32_t g0 = blockIdx.x * STEP + threadIdx.x; g0 < p.n_total; g0 += gridDim.x * STEP) {
        uint32_t g[kExtractEPT], r[kExtractEPT], i[kExtractEPT], ks[kExtractEPT], fs[kExtractEPT];
        uint64_t off[kExtractEPT], expect[kExtractEPT], dlen_total[kExtractEPT];
        const uint8_t *data[kExtractEPT];
        bool act[kExtractEPT], ok[kExtractEPT];
        uint4 c_rec[kExtractEPT], c_pr[kExtractEPT];
        if (kPersist) {
#pragma unroll
            for (int u = 0; u < kExtractEPT; u++) { c_rec[u] = n_rec[u]; c_pr[u] = n_pr[u]; r[u] = n_run[u]; }
            fetch((uint64_t)g0 + (uint64_t)gridDim.x * STEP, n_rec, n_pr, n_run); // travels while this step's headers do
        } else {
            fetch(g0, c_rec, c_pr, r);
        }
        // ---- phase 1: what the index records say
#pragma unroll
        for (int u = 0; u < kExtractEPT; u++) {
            g[u] = g0 + u * 256u;
            act[u] = g[u] < p.n_total;
            ok[u] = false;
            if (!act[u]) continue;
            const RunDesc &rd = p.runs[r[u]];
            i[u] = g[u] - rd.base;
            data[u] = rd.data;
            dlen_total[u] = rd.data_len;
            const uint4 rec = c_rec[u];
            off[u] = (uint64_t)rec.x | ((uint64_t)rec.y << 32);
            ks[u] = rec.z;
            fs[u] = rec.w;
            expect[u] = rd.off_base;
            if (i[u] && !redo) {
                const uint4 pr = c_pr[u];
                expect[u] = ((uint64_t)pr.x | ((uint64_t)pr.y << 32)) + pr.w;
            }
        }
        // ---- phase 2: everything that can be decided from the index alone, then the entry header loads
        uint64_t klen_w[kExtractEPT], dlen_w[kExtractEPT], w0[kExtractEPT], w1[kExtractEPT];
        uint64_t ts_lo[kExtractEPT], ts_hi[kExtractEPT];
        bool match[kExtractEPT];
#pragma unroll
        for (int u = 0; u < kExtractEPT; u++) {
            if (!act[u]) continue;
            if (redo) {
                ok[u] = i[u] < p.first_bad[r[u]];
            } else {
                ok[u] = ks[u] >= 8 && (uint64_t)fs[u] >= (uint64_t)ks[u] + 24 && off[u] <= dlen_total[u] &&
                        (uint64_t)fs[u] <= dlen_total[u] - off[u] && (off[u] == expect[u] || p.sparse_offsets);
            }
            match[u] = false;
            klen_w[u] = dlen_w[u] = w0[u] = w1[u] = 0;
            ts_lo[u] = ts_hi[u] = 0;
            if (ok[u]) {
                const uint8_t *e = data[u] + off[u];
                klen_w[u] = ldu(e);
                dlen_w[u] = ldu(e + ks[u]);
                if (kRef && !redo) {
                    ts_lo[u] = ldu(e + fs[u] - 16);
                    ts_hi[u] = ldu(e + fs[u] - 8);
                }
                const uint32_t klen = ks[u] - 8;
                match[u] = klen >= L;
                if (match[u]) {
                    const uint8_t *key = e + 8;
                    // every load below stays inside the entry: >= 24 bytes (dlen + timestamp) follow the key
                    w0[u] = ldu(key + L);
                    w1[u] = ldu(key + L + 8);
                    for (uint32_t q = 0; q < npw; q++) {
                        const uint64_t kw = ldu(key + 8 * q);
                        const uint32_t nb = L - 8 * q; // prefix bytes in this word (>= 1)
                        const uint64_t mask = nb >= 8 ? ~0ull : ((1ull << (8 * nb)) - 1);
                        match[u] = match[u] && (((kw ^ pfx[q]) & mask) == 0);
                    }
                }
            }
        }
        // ---- phase 3: verdicts and records
#pragma unroll
        for (int u = 0; u < kExtractEPT; u++) {
            if (!act[u]) continue;
            if (!redo) {
                if (ok[u]) ok[u] = klen_w[u] == (uint64_t)(ks[u] - 8) && dlen_w[u] == (uint64_t)(fs[u] - ks[u] - 24);
                if (kRef) {
                    // hi == 0 covers every non-negative count below 2^64 ns (year 2554): in range without the division
                    if (ok[u] && ts_hi[u] != 0) ok[u] = ts_decodes(ts_lo[u], ts_hi[u]);
                    // Anything wrong in pass 0 may be the index's fault rather than the data's: only the canonical index
                    // can tell, so note it (cheap: the flag is set at most once per bad record).  Pass 2 is final.
                    if (!ok[u] && mode == 0) atomicOr(&c->flags, kFlagIndexDiffers);
                }
                if (!ok[u]) {
                    atomicMin(&p.first_bad[r[u]], i[u]);
                    atomicOr(&c->flags, kFlagTruncated);
                }
            }
            Rec out;
            out.x = out.y = out.z = 0;
            out.w = g[u];
            if (ok[u]) {
                if (match[u]) out = make_rec(w0[u], w1[u], (uint64_t)(ks[u] - 8 - L), g[u]);
                else atomicMin(&p.first_mismatch[r[u]], i[u]);
            }
            st_rec(&p.rec_a[g[u]], out);
        }
        // ---- bloom hashes, here rather than in the gather: this kernel waits on memory with its issue slots idle, the key
        // bytes are in L1, and the gather is the kernel that has no instruction to spare (DESIGN.md section 5, K1 / K5)
        if (kHash && !redo && p.hash_rec != nullptr) {
#pragma unroll
            for (int u = 0; u < kExtractEPT; u++) {
                if (!act[u] || !ok[u]) continue;
                const uint8_t *key = data[u] + off[u] + 8;
                uint64_t h0, h1;
                sip13_pair_vec_u8(p.bloom.sip, (uint64_t)(ks[u] - 8), [key](uint64_t q) { return ld_u64_unaligned(key + 8 * q); }, &h0, &h1);
                p.hash_rec[g[u]] = make_uint4((uint32_t)h0, (uint32_t)(h0 >> 32), (uint32_t)h1, (uint32_t)(h1 >> 32));
            }
        }
    }
}

__device__ __forceinline__ void block_excl_scan_1024(unsigned long long &vb, uint32_t &vc, unsigned long long *s_b, uint32_t *s_c,
                                                     unsigned long long *tot_b, uint32_t *tot_c);

// ------------------------------------------------------------------------------------
// K1b: per-run valid counts -> segment tables of every merge level (one CTA of 1024 threads).

__global__ void __launch_bounds__(1024) k_plan(Params p) {
    pdl_trigger();
    pdl_wait();
    // One CTA: level-0 segments in parallel, then level after level (segment l+1 = a pair of level l; the exclusive scan of
    // the pairs' tile counts is a block scan carried over chunks of 1024 pairs).  Batches hold up to 2^24 leaf segments.
    __shared__ unsigned long long s_b[32];
    __shared__ uint32_t s_c[32];
    __shared__ uint32_t s_total, s_trunc, s_flags;
    Ctl *c = p.ctl;
    const uint32_t tid = threadIdx.x;
    if (tid == 0) { s_total = 0; s_trunc = 0; s_flags = 0; }
    __syncthreads();
    uint32_t total = 0, trunc = 0, flags = 0;
    if (p.mode_flush) {
        // arrival batches: level-0 segments are the tiles k_block_sort leaves sorted.  With several memtables
        // (flush-many) each one owns an aligned block of `slots` leaf segments, so the first log2(slots) merge
        // levels never pair segments of different memtables -- and there are no further levels.
        const uint32_t slots = p.flush_slots ? p.flush_slots : p.nseg[0];
        const uint64_t n_leaf = (uint64_t)p.n_runs * slots;
        for (uint64_t k = tid; k < n_leaf; k += 1024) {
            const uint32_t m = (uint32_t)(k / slots), j = (uint32_t)(k % slots);
            const uint32_t cnt = p.first_bad[m];
            const uint32_t s0 = j * (uint32_t)kMergeTile;
            Seg sg;
            sg.start = p.runs[m].base + s0;
            sg.len = cnt > s0 ? (cnt - s0 < (uint32_t)kMergeTile ? cnt - s0 : (uint32_t)kMergeTile) : 0;
            p.seg[0][k] = sg;
            if (j == 0) {
                total += cnt;
                if (cnt < p.runs[m].n_in) trunc++;
            }
        }
    } else if (p.group_slots) {
        // compact-many: job g's runs fill the first slots of its block, the rest are empty segments parked at its end
        const uint64_t n_leaf = (uint64_t)p.n_groups * p.group_slots;
        for (uint64_t k = tid; k < n_leaf; k += 1024) {
            const uint32_t g = (uint32_t)(k / p.group_slots), sl = (uint32_t)(k % p.group_slots);
            const GroupDesc &gd = p.groups[g];
            Seg sg;
            sg.start = gd.pos_end;
            sg.len = 0;
            if (sl < gd.n_runs) {
                const uint32_t r = gd.first_run + sl;
                const uint32_t cnt = p.first_bad[r];
                if (cnt < p.runs[r].n_in) trunc++;
                if (p.first_mismatch[r] < cnt) flags |= kFlagUnsorted;
                sg.start = p.runs[r].base;
                sg.len = cnt;
                total += cnt;
            }
            p.seg[0][k] = sg;
        }
    } else {
        for (uint32_t r = tid; r < p.n_runs; r += 1024) {
            const uint32_t cnt = p.first_bad[r];
            if (cnt < p.runs[r].n_in) trunc++;
            if (p.first_mismatch[r] < cnt) flags |= kFlagUnsorted;
            p.seg[0][r].start = p.runs[r].base;
            p.seg[0][r].len = cnt;
            total += cnt;
        }
    }
    if (total) atomicAdd(&s_total, total);
    if (trunc) atomicAdd(&s_trunc, trunc);
    if (flags) atomicOr(&s_flags, flags);
    __syncthreads();
    for (uint32_t l = 0; l < p.n_levels; l++) {
        const uint32_t pairs = p.nseg[l + 1];
        uint32_t carry = 0;
        for (uint32_t j0 = 0; j0 < pairs; j0 += 1024) {
            const uint32_t j = j0 + tid;
            uint32_t tiles = 0;
            if (j < pairs) {
                const Seg a = p.seg[l][2 * j];
                const uint32_t blen = (2 * j + 1 < p.nseg[l]) ? p.seg[l][2 * j + 1].len : 0;
                p.seg[l + 1][j].start = a.start;
                p.seg[l + 1][j].len = a.len + blen;
                const uint32_t tl = (p.fin_tile && l + 1 == p.n_levels) ? p.fin_tile : (uint32_t)kMergeTile;
                tiles = (a.len + blen + tl - 1) / tl;
            }
            unsigned long long vb = 0, tb;
            uint32_t vc = tiles, tc;
            __syncthreads();
            block_excl_scan_1024(vb, vc, s_b, s_c, &tb, &tc);
            if (j < pairs) p.tile_base[l][j] = carry + vc;
            carry += tc;
        }
        if (tid == 0) p.tile_base[l][pairs] = carry;
        __syncthreads(); // seg[l + 1] complete before the next level pairs it up
    }
    if (tid == 0) {
        c->total = s_total;
        c->span = p.n_groups ? p.n_total : s_total; // groups keep their slices at their input positions: gaps stay
        c->runs_truncated = s_trunc;
        c->flags = c->flags | s_flags;
    }
}

// ------------------------------------------------------------------------------------
// Flush (memtable) front end.  An arrival batch is not sorted, so the common prefix is the
// minimum over ALL keys of their common prefix with arrival 0, and the level-0 segments are
// produced by an in-CTA merge sort of kMergeTile-record (1792) tiles ordered by (key, arrival).

__global__ void k_flush_prefix_init(Params p) {
    pdl_trigger();
    pdl_wait();
    if (threadIdx.x || blockIdx.x) return;
    Ctl *c = p.ctl;
    const uint8_t *ptr;
    uint32_t kl = 0;
    uint32_t L = 0;
    const RunDesc &rd = p.runs[p.flush_ref_run];
    if (rd.n_in && safe_key(rd, 0, &ptr, &kl)) {
        L = kl < kMaxPrefix ? kl : kMaxPrefix;
        for (uint32_t i = 0; i < L; i++) c->prefix[i] = __ldg(ptr + i);
    }
    c->prefix_len = L;
}

__global__ void __launch_bounds__(256) k_flush_prefix(Params p) {
    pdl_trigger();
    pdl_wait();
    Ctl *c = p.ctl;
    uint32_t g = blockIdx.x * 256u + threadIdx.x;
    uint32_t L = c->prefix_len; // only ever shrinks; a stale (larger) value is still an upper bound
    if (g < p.n_total && L) {
        const uint32_t r = find_run(p, g);
        const uint8_t *ptr;
        uint32_t kl;
        if (safe_key(p.runs[r], g - p.runs[r].base, &ptr, &kl)) {
            uint32_t m = kl < L ? kl : L, i = 0;
            while (i < m && __ldg(ptr + i) == c->prefix[i]) i++;
            L = i;
        }
        // an unreadable record is cut off by validation later; it must not widen the window
    }
    for (int o = 16; o; o >>= 1) {
        uint32_t other = __shfl_xor_sync(0xFFFFFFFFu, L, o);
        L = other < L ? other : L;
    }
    if ((threadIdx.x & 31) == 0 && L < c->prefix_len) atomicMin(&c->prefix_len, L);
}

// total order for sorting arrivals: key, then arrival index (= gid)
__device__ __forceinline__ bool arrival_less(const Params &p, uint32_t skip, const Rec &a, const Rec &b) {
    int und;
    int c = rec_cmp_window(a, b, &und);
    if (und) c = full_key_cmp(p, a.w, b.w, skip);
    return c < 0 || (c == 0 && a.w < b.w);
}

__global__ void __launch_bounds__(kMergeThreads) k_block_sort(Params p) {
    pdl_trigger();
    pdl_wait();
    __shared__ Rec s[kMergeTile + kMergeVT + 1];
    const Seg sg = p.seg[0][blockIdx.x]; // the tile this CTA sorts (k_plan)
    const uint32_t base = sg.start;
    const uint32_t n = sg.len;
    if (n == 0) return;
    const uint32_t tid = threadIdx.x;
    const uint32_t skip = p.ctl->prefix_len + kWindowBytes;
    Rec inf;
    inf.x = inf.y = inf.z = inf.w = 0xFFFFFFFFu; // clamp byte 0xFF: above every real record, never "undecided"
    for (uint32_t i = tid; i < (uint32_t)kMergeTile; i += kMergeThreads) s[i] = i < n ? ld_rec(&p.rec_a[base + i]) : inf;
    __syncthreads();
    Rec r[kMergeVT];
#pragma unroll
    for (int i = 0; i < kMergeVT; i++) r[i] = s[tid * kMergeVT + i];
    // odd-even transposition sort of the thread's 8 records
#pragma unroll
    for (int pass = 0; pass < kMergeVT; pass++) {
#pragma unroll
        for (int i = pass & 1; i + 1 < kMergeVT; i += 2) {
            if (arrival_less(p, skip, r[i + 1], r[i])) { Rec t = r[i]; r[i] = r[i + 1]; r[i + 1] = t; }
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kMergeVT; i++) s[tid * kMergeVT + i] = r[i];
    __syncthreads();
    for (uint32_t len = kMergeVT; len < (uint32_t)kMergeTile; len <<= 1) {
        const uint32_t d0 = tid * kMergeVT;
        const uint32_t pair = d0 / (2 * len);
        const uint32_t diag = d0 - pair * 2 * len;
        const Rec *A = s + pair * 2 * len;
        const Rec *B = A + len;
        uint32_t lo = diag > len ? diag - len : 0;
        uint32_t hi = diag < len ? diag : len;
        while (lo < hi) {
            uint32_t mid = (lo + hi) >> 1;
            if (!arrival_less(p, skip, B[diag - 1 - mid], A[mid])) lo = mid + 1; else hi = mid;
        }
        uint32_t ai = lo, bi = diag - lo;
        Rec ak = A[ai < len ? ai : len - 1], bk = B[bi < len ? bi : len - 1];
#pragma unroll
        for (int i = 0; i < kMergeVT; i++) {
            bool has_a = ai < len, has_b = bi < len;
            bool take_b = has_b && (!has_a || arrival_less(p, skip, bk, ak));
            r[i] = take_b ? bk : ak;
            if (take_b) { bi++; if (bi < len) bk = B[bi]; } else { ai++; if (ai < len) ak = A[ai]; }
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < kMergeVT; i++) s[d0 + i] = r[i];
        __syncthreads();
    }
    for (uint32_t i = tid; i < n; i += kMergeThreads) st_rec(&p.rec_a[base + i], s[i]);
}

// ------------------------------------------------------------------------------------
// K2/K3: one merge level = merge-path partition + tile merge.  Pair j of level l merges
// segments 2j (A) and 2j+1 (B) of `src` into one segment of `dst` starting at A.start.
// A holds lower run positions than B, and ties take A first, so equal keys stay ordered by
// run position (= gid) through every level.

__device__ __forceinline__ uint32_t find_pair(const uint32_t *tb, uint32_t pairs, uint32_t v, uint32_t slope) {
    // largest j in [0, pairs) with tb[j] + slope * j <= v
    uint32_t lo = 0, hi = pairs;
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (tb[mid] + slope * mid <= v) lo = mid; else hi = mid;
    }
    return lo;
}

// One WARP per tile boundary: the merge-path search is a 32-ary search (32 probes of the diagonal per round,
// one ballot), 5 rounds for a 4M-record diagonal instead of 22 dependent global-memory round trips.
constexpr int kPartitionThreads = 256;

__global__ void __launch_bounds__(kPartitionThreads) k_merge_partition(const __grid_constant__ Params p, uint32_t level, const Rec *src) {
    pdl_trigger();
    pdl_wait();
    const uint32_t pairs = p.nseg[level + 1];
    const uint32_t *tb = p.tile_base[level];
    const uint32_t n_bound = tb[pairs] + pairs; // every pair has tiles + 1 boundaries
    const uint32_t idx = (blockIdx.x * (uint32_t)kPartitionThreads + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (idx >= n_bound) return; // warp-uniform
    const uint32_t skip = p.ctl->prefix_len + kWindowBytes;
    uint32_t j = find_pair(tb, pairs, idx, 1);
    uint32_t t = idx - (tb[j] + j);
    Seg a = p.seg[level][2 * j];
    Seg b;
    b.start = 0; b.len = 0;
    if (2 * j + 1 < p.nseg[level]) b = p.seg[level][2 * j + 1];
    const bool fin = p.fin_tile && level + 1 == p.n_levels;
    uint64_t d64 = (uint64_t)t * (fin ? p.fin_tile : (uint32_t)kMergeTile);
    uint32_t n = a.len + b.len;
    uint32_t diag = d64 < n ? (uint32_t)d64 : n;
    uint32_t lo = diag > b.len ? diag - b.len : 0;
    uint32_t hi = diag < a.len ? diag : a.len;
    // P(mid) = "B[diag-1-mid] is not less than A[mid]" is true for mid < answer and false from the answer on
    while (lo < hi) {
        const uint32_t range = hi - lo;
        const uint32_t step = range >= 32 ? range >> 5 : 1;
        const uint32_t mid = lo + lane * step + (step - 1); // ascending in the lane; < hi for every lane when range >= 32
        bool pr = false;
        if (mid < hi) {
            Rec ra = ld_rec(&src[a.start + mid]);
            Rec rb = ld_rec(&src[b.start + (diag - 1 - mid)]);
            pr = !key_less(p, skip, rb, ra);
        }
        const uint32_t cnt = __popc(__ballot_sync(0xFFFFFFFFu, pr)); // P is monotone: the true probes are lanes 0..cnt-1
        const uint32_t first_false = lo + cnt * step + (step - 1);     // probe of lane cnt (if it exists and is < hi)
        lo = lo + cnt * step;
        if (cnt < 32 && first_false < hi) hi = first_false;
        else if (range < 32) hi = lo; // every valid probe was true: the answer is the end of the range
    }
    if (lane == 0) {
        p.part[idx] = lo;
        // everything a merge tile needs, one record per boundary: the persistent merge kernels read two of them per tile
        // (one round trip, issued a tile ahead) instead of walking tile_base / seg / part (five dependent ones)
        if (!fin) p.bnd[idx] = make_uint4(a.start + lo, b.start + (diag - lo), a.start + diag, j);
        if (t * (uint64_t)(fin ? p.fin_tile : (uint32_t)kMergeTile) < n) p.tile_bnd[tb[j] + t] = idx; // a tile starts here
    }
    if (fin) {
        // k_merge_final: a group of equal keys must not straddle a tile border, or the head's thread would have to walk the
        // rest of the group through global memory while its whole CTA (and, through the chained scan, every later tile)
        // waits.  So the border moves forward past the records that carry the key of the last record before it: up to 31
        // of A and 31 of B (more only with hundreds of runs holding one key: then the kernel's walk does the rest).
        uint32_t ext = 0;
        if (diag > 0 && diag < n) {
            const uint32_t ai = lo, bi = diag - lo;
            Rec K;
            if (ai == 0) K = ld_rec(&src[b.start + bi - 1]);
            else if (bi == 0) K = ld_rec(&src[a.start + ai - 1]);
            else {
                const Rec ka = ld_rec(&src[a.start + ai - 1]), kb = ld_rec(&src[b.start + bi - 1]);
                K = key_less(p, skip, ka, kb) ? kb : ka;
            }
            const bool ea = ai + lane < a.len && key_equal(p, skip, K, ld_rec(&src[a.start + ai + lane]));
            const bool eb = bi + lane < b.len && key_equal(p, skip, K, ld_rec(&src[b.start + bi + lane]));
            const uint32_t ma = __ballot_sync(0xFFFFFFFFu, ea), mb = __ballot_sync(0xFFFFFFFFu, eb);
            uint32_t xa = (uint32_t)__ffs((int)~ma), xb = (uint32_t)__ffs((int)~mb); // 1 + leading run of equal records; 0 = all 32
            xa = xa ? xa - 1 : 32;
            xb = xb ? xb - 1 : 32;
            ext = (xa > 31 ? 31u : xa) | ((xb > 31 ? 31u : xb) << 8);
        }
        if (lane == 0) {
            p.part_ext[idx] = ext;
            p.bnd[idx] = make_uint4(a.start + lo + (ext & 0xFF), b.start + (diag - lo) + (ext >> 8), a.start + diag, j);
        }
    }
}

__global__ void __launch_bounds__(kMergeThreads, 4) k_merge(Params p, uint32_t level, const Rec *src, Rec *dst) {
    pdl_trigger();
    pdl_wait();
    __shared__ Rec s[kMergeTile + kMergeVT + 1];
    const uint32_t pairs = p.nseg[level + 1];
    const uint32_t *tb = p.tile_base[level];
    const uint32_t tile = blockIdx.x;
    if (tile >= tb[pairs]) return;
    const uint32_t tid = threadIdx.x;
    const uint32_t skip = p.ctl->prefix_len + kWindowBytes;
    uint32_t j = find_pair(tb, pairs, tile, 0);
    uint32_t t = tile - tb[j];
    Seg a = p.seg[level][2 * j];
    Seg b;
    b.start = 0; b.len = 0;
    if (2 * j + 1 < p.nseg[level]) b = p.seg[level][2 * j + 1];
    const uint32_t pidx = tb[j] + j + t;
    const uint32_t a0 = p.part[pidx], a1 = p.part[pidx + 1];
    const uint32_t total = a.len + b.len;
    const uint32_t diag0 = t * kMergeTile;
    const uint32_t diag1 = diag0 + kMergeTile < total ? diag0 + kMergeTile : total;
    const uint32_t b0 = diag0 - a0, b1 = diag1 - a1;
    const uint32_t nA = a1 - a0, nB = b1 - b0, n = nA + nB;

    for (uint32_t i = tid; i < nA; i += kMergeThreads) s[i] = ld_rec(&src[a.start + a0 + i]);
    for (uint32_t i = tid; i < nB; i += kMergeThreads) s[nA + i] = ld_rec(&src[b.start + b0 + i]);
    __syncthreads();

    uint32_t d = tid * kMergeVT;
    if (d > n) d = n;
    uint32_t lo = d > nB ? d - nB : 0;
    uint32_t hi = d < nA ? d : nA;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (!key_less_smem(p, skip, &s[nA + d - 1 - mid], &s[mid])) lo = mid + 1; else hi = mid;
    }
    uint32_t ai = lo, bi = d - lo;
    Rec ak = s[ai], bk = s[nA + bi]; // may read one slot past a range: slack + guarded below
    Rec out[kMergeVT];
#pragma unroll
    for (int i = 0; i < kMergeVT; i++) {
        bool has_a = ai < nA, has_b = bi < nB;
        bool take_b = has_b && (!has_a || key_less(p, skip, bk, ak));
        out[i] = take_b ? bk : ak;
        if (take_b) { bi++; bk = s[nA + bi]; } else { ai++; ak = s[ai]; }
    }
    Rec *o = dst + a.start + diag0;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kMergeVT; i++)
        if (d + i < n) s[d + i] = out[i];
    __syncthreads();
    for (uint32_t i = tid; i < n; i += kMergeThreads) st_rec(&o[i], s[i]);
}

// ------------------------------------------------------------------------------------
// Tile descriptors for the persistent merge kernel: which records of src a tile consumes and where
// its merged output goes.  Looked up two tiles ahead so the lookups never sit on the critical path.

struct MergeDesc {
    uint32_t a_src, n_a, b_src, n_b, dst; // record offsets into src / dst, counts
};

__device__ __forceinline__ MergeDesc merge_desc(const Params &p, uint32_t level, uint32_t tile) {
    const uint32_t pairs = p.nseg[level + 1];
    const uint32_t *tb = p.tile_base[level];
    MergeDesc d;
    d.a_src = d.n_a = d.b_src = d.n_b = d.dst = 0;
    if (tile >= tb[pairs]) return d;
    const uint32_t j = find_pair(tb, pairs, tile, 0);
    const uint32_t t = tile - tb[j];
    const Seg a = p.seg[level][2 * j];
    Seg b;
    b.start = 0; b.len = 0;
    if (2 * j + 1 < p.nseg[level]) b = p.seg[level][2 * j + 1];
    const uint32_t pidx = tb[j] + j + t;
    const uint32_t a0 = p.part[pidx], a1 = p.part[pidx + 1];
    const uint32_t total = a.len + b.len;
    const uint32_t diag0 = t * kMergeTile;
    const uint32_t diag1 = diag0 + kMergeTile < total ? diag0 + kMergeTile : total;
    d.a_src = a.start + a0;
    d.n_a = a1 - a0;
    d.b_src = b.start + (diag0 - a0);
    d.n_b = (diag1 - a1) - (diag0 - a0);
    d.dst = a.start + diag0;
    return d;
}

constexpr int kMergeBufRecs = kMergeTile + kMergeVT + 1;

// ------------------------------------------------------------------------------------
// K3 (TMA variant): the merge tiles are the one place on this path where data IS a 16-byte-aligned
// contiguous block (fixed-size records), so the tile's A range and B range come in as two
// cp.async.bulk (TMA, 1-D) copies completing on an mbarrier, and the merged tile leaves as one
// bulk store -- no per-thread global loads or stores at all.  Persistent CTAs, two shared-memory
// buffers: tile q+1 lands while tile q is searched and merged.

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_1d(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(kMergeThreads, kMergeCtasPerSM) k_merge_tma(const __grid_constant__ Params p, uint32_t level, const Rec *src, Rec *dst) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(128) uint8_t s_raw[];
    Rec *bufs[2] = {reinterpret_cast<Rec *>(s_raw), reinterpret_cast<Rec *>(s_raw) + kMergeBufRecs};
    __shared__ __align__(8) uint64_t s_bar[2];
    const uint32_t tid = threadIdx.x;
    const uint32_t skip = p.ctl->prefix_len + kWindowBytes;
    const uint32_t n_tiles = p.tile_base[level][p.nseg[level + 1]];
    const uint32_t G = gridDim.x;
    uint32_t tile = blockIdx.x;
    if (tile >= n_tiles) return;
    if (tid == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto issue = [&](const MergeDesc &d, Rec *buf, uint64_t *bar) { // thread 0 only
        mbar_expect_tx(bar, (d.n_a + d.n_b) * 16u);
        if (d.n_a) tma_load_1d(buf, &src[d.a_src], d.n_a * 16u, bar);
        if (d.n_b) tma_load_1d(buf + d.n_a, &src[d.b_src], d.n_b * 16u, bar);
    };

    // Tile descriptors from the boundary records k_merge_partition left: tile -> boundary index (one load, issued three tiles
    // ahead), then the two boundary records (two loads, issued two tiles ahead): no dependent chain inside an iteration.
    auto ld_bidx = [&](uint32_t t) -> uint32_t { return t < n_tiles ? __ldg(&p.tile_bnd[t]) : 0xFFFFFFFFu; };
    auto mk_desc = [&](uint32_t bidx) -> MergeDesc {
        MergeDesc d;
        d.a_src = d.n_a = d.b_src = d.n_b = d.dst = 0;
        if (bidx == 0xFFFFFFFFu) return d;
        const uint4 b0 = __ldg(&p.bnd[bidx]), b1 = __ldg(&p.bnd[bidx + 1]);
        d.a_src = b0.x; d.n_a = b1.x - b0.x;
        d.b_src = b0.y; d.n_b = b1.y - b0.y;
        d.dst = b0.z;
        return d;
    };
    MergeDesc cur = mk_desc(ld_bidx(tile));
    MergeDesc nxt = mk_desc(ld_bidx(tile + G));
    uint32_t bidx2 = ld_bidx(tile + 2 * G);
    if (tid == 0) issue(cur, bufs[0], &s_bar[0]);
    for (uint32_t q = 0;; q++) {
        Rec *s = bufs[q & 1];
        const bool has_next = tile + G < n_tiles;
        if (tid == 0 && has_next) {
            // buffer (q+1)&1 staged tile q-1's output: its bulk store must have finished READING it
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            issue(nxt, bufs[(q + 1) & 1], &s_bar[(q + 1) & 1]);
        }
        const MergeDesc nn = mk_desc(bidx2);           // consumed one iteration from now
        const uint32_t bidx3 = ld_bidx(tile + 3 * G);  // ... and two iterations from now
        while (!mbar_try_wait(&s_bar[q & 1], (q >> 1) & 1)) {}

        const uint32_t nA = cur.n_a, nB = cur.n_b, n = nA + nB;
        uint32_t d = tid * kMergeVT;
        if (d > n) d = n;
        uint32_t lo = d > nB ? d - nB : 0;
        uint32_t hi = d < nA ? d : nA;
        while (lo < hi) {
            uint32_t mid = (lo + hi) >> 1;
            if (!key_less_smem(p, skip, &s[nA + d - 1 - mid], &s[mid])) lo = mid + 1; else hi = mid;
        }
        uint32_t ai = lo, bi = d - lo;
        Rec ak = s[ai], bk = s[nA + bi];
        Rec out[kMergeVT];
#pragma unroll
        for (int i = 0; i < kMergeVT; i++) {
            bool has_a = ai < nA, has_b = bi < nB;
            bool take_b = has_b && (!has_a || key_less(p, skip, bk, ak));
            out[i] = take_b ? bk : ak;
            if (take_b) { bi++; bk = s[nA + bi]; } else { ai++; ak = s[ai]; }
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < kMergeVT; i++)
            if (d + i < n) s[d + i] = out[i];
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // generic-proxy writes -> visible to the bulk store
        __syncthreads();
        if (tid == 0) {
            tma_store_1d(dst + cur.dst, s, n * 16u);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        if (!has_next) break;
        tile += G;
        cur = nxt;
        nxt = nn;
        bidx2 = bidx3;
    }
    if (tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); // stores complete before the CTA retires
}

// ------------------------------------------------------------------------------------
// K4a: resolve.  One thread per merged record, no ordering between CTAs.
//
// A record that starts a group of equal keys ("head") picks the group's winner -- the entry
// with the greatest (timestamp, run position), lsm_tree.rs:1041-1044 with mod.rs:75-81 and
// lsm_tree.rs:58-65 -- and emits it unless it is a tombstone that must go
// (lsm_tree.rs:1045-1046).  Every thread fetches its own entry's index record, and -- only if
// it sits in a group of two or more -- its own timestamp, so the loads of a group run in
// parallel; the head then reduces over shared memory.
// Output, in merged order: res[i] = {entry address (u64), key_size, full_size or 0 if nothing
// is emitted at position i}, plus each 256-record tile's (bytes, entries) aggregate.

__device__ __forceinline__ void ld_ts(const uint8_t *entry, uint32_t full_size, uint64_t *lo, uint64_t *hi) {
    const uint8_t *t = entry + full_size - 16;
    *lo = ld_u64_unaligned(t);
    *hi = ld_u64_unaligned(t + 8);
}

#ifndef DBEEL_RESOLVE_MINB
#define DBEEL_RESOLVE_MINB 14 // 14 CTAs of 128 threads per SM = a 36-register cap
#endif
constexpr unsigned long long kScanAgg = 1, kScanPrefix = 2; // 0 = nothing published yet

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long *q) {
    unsigned long long v;
    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(q) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_u64(unsigned long long *q, unsigned long long v) {
    asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(q), "l"(v) : "memory");
}

// kFused: the offsets scan and k_emit's writes happen here too -- every tile publishes its (bytes, entries) aggregate, looks
// back over its predecessors' aggregates / inclusive prefixes (one warp, 32 predecessors per step) and writes its survivors'
// .index records, source addresses and gather-tile markers directly.  Saves the res[] round trip (2 x 16 B per merged
// record), two scan kernels and k_emit's launch.  Single jobs only: the grouped paths cut the stream by res[] afterwards.
#ifndef DBEEL_RESOLVE_FUSED_MINB
#define DBEEL_RESOLVE_FUSED_MINB 12
#endif
template <bool kNarrow, bool kFused, bool kHashRec>
__global__ void __launch_bounds__(kResolveThreads, kFused ? DBEEL_RESOLVE_FUSED_MINB : DBEEL_RESOLVE_MINB) k_resolve(Params p, const Rec *m, uint4 *res) {
    pdl_trigger();
    pdl_wait();
    constexpr int NT = kResolveThreads;
    __shared__ Rec s_rec[NT + 2];
    __shared__ unsigned long long s_entry[NT]; // device address of each record's entry
    __shared__ uint32_t s_ks[NT], s_fs[NT];
    __shared__ unsigned long long s_tlo[NT], s_thi[NT];
    __shared__ uint8_t s_eqn[NT]; // record tid has the same key as record tid+1
    const Ctl *c = p.ctl;
    const uint32_t tid = threadIdx.x;
    const uint32_t span = c->span;
    __shared__ uint32_t s_tile;
    if (kFused) { // tiles numbered by starting order: a tile only ever waits for tiles that are already running
        if (tid == 0) s_tile = atomicAdd(p.scan_ticket, 1u);
        __syncthreads();
    }
    const uint32_t tile_id = kFused ? s_tile : blockIdx.x;
    const uint32_t i0 = tile_id * NT;
    if (i0 >= span) return;
    const uint32_t skip = c->prefix_len + kWindowBytes;
    const uint32_t i = i0 + tid;
    // the sorted segment position i belongs to: the whole merged array, or -- flush-many -- one memtable's slice
    uint32_t lim_lo = 0, lim_hi = c->total;
    int keep_tombstones = p.keep_tombstones;
    if (p.n_groups && i < span) {
        const uint32_t g = find_group(p, i);
        const Seg sl = p.seg[p.n_levels][g];
        lim_lo = sl.start;
        lim_hi = sl.start + sl.len;
        if (p.groups) keep_tombstones = p.groups[g].keep_tombstones;
    }

    // records i0-1 .. i0+NT (coalesced), so neighbours come from shared memory
    for (uint32_t k = tid; k < NT + 2; k += NT) {
        int64_t gi = (int64_t)i0 - 1 + k;
        if (gi >= 0 && gi < (int64_t)span) s_rec[k] = ld_rec(&m[gi]);
    }
    __syncthreads();

    const bool active = i < span && i < lim_hi;
    bool eq_prev = false, eq_next = false;
    Rec cur;
    cur.x = cur.y = cur.z = cur.w = 0;
    KeyRef me;
    me.entry = nullptr; me.ptr = nullptr; me.klen = 0; me.full_size = 0;
    if (active) {
        cur = s_rec[tid + 1];
        if (i > lim_lo) eq_prev = key_equal(p, skip, s_rec[tid], cur);
        if (i + 1 < lim_hi) eq_next = key_equal(p, skip, cur, s_rec[tid + 2]);
        if (kNarrow) {
            const uint32_t r = find_run(p, cur.w);
            const RunDesc &rd = p.runs[r];
            const uint4 rec = ldg128_narrow(&rd.index[cur.w - rd.base]);
            me.entry = rd.data + ((uint64_t)rec.x | ((uint64_t)rec.y << 32));
            me.ptr = me.entry + 8;
            me.klen = rec.z - 8;
            me.full_size = rec.w;
        } else {
            me = key_of_gid(p, cur.w);
        }
        uint64_t tlo = 0, thi = 0;
        if ((eq_prev || eq_next) && !p.mode_flush) {
            if (kNarrow) {
                const uint8_t *t = me.entry + me.full_size - 16;
                tlo = ld_u64_unaligned_narrow(t);
                thi = ld_u64_unaligned_narrow(t + 8);
            } else {
                ld_ts(me.entry, me.full_size, &tlo, &thi);
            }
        }
        s_tlo[tid] = tlo;
        s_thi[tid] = thi;
    }
    s_entry[tid] = (unsigned long long)(uintptr_t)me.entry;
    s_ks[tid] = me.klen + 8;
    s_fs[tid] = me.full_size;
    s_eqn[tid] = eq_next ? 1 : 0;
    __syncthreads();

    uint32_t keep = 0, ks = 0, fs = 0, wgid = 0;
    unsigned long long src = 0;
    if (p.mode_flush) {
        // Arrival batches: the winner of a group of equal keys is simply its LAST member (RedBlackTree::set replaces in place,
        // lib.rs:509-511), and every member knows locally whether it is the last one.  No walk over the group: a hot key of a
        // Zipf stream fills hundreds of consecutive positions of a memtable, and a head thread stepping through them one
        // dependent load at a time dominated the whole flush of a Zipf stream.
        if (active && !eq_next) {
            keep = 1; // tombstones are ordinary entries of a flush (lsm_tree.rs:790-795)
            ks = s_ks[tid]; fs = s_fs[tid]; src = s_entry[tid];
            wgid = cur.w;
        }
    } else if (active && !eq_prev) { // head of its group
        uint32_t w = tid; // winner so far, as an index into this tile's shared arrays
        ks = s_ks[tid]; fs = s_fs[tid]; src = s_entry[tid];
        wgid = cur.w;
        if (eq_next) {
            uint64_t wlo = s_tlo[tid], whi = s_thi[tid];
            uint32_t j = tid;
            bool more = true;
            while (more && j + 1 < NT) { // members inside the tile
                j++;
                // the later member wins ties: it comes from a later run position (larger gid);
                // in flush mode the later arrival always wins (lib.rs:509-511)
                bool better = p.mode_flush || !ts_greater(wlo, whi, s_tlo[j], s_thi[j]);
                if (better) { w = j; wlo = s_tlo[j]; whi = s_thi[j]; }
                more = s_eqn[j] != 0;
            }
            ks = s_ks[w]; fs = s_fs[w]; src = s_entry[w];
            wgid = s_rec[w + 1].w;
            if (more) { // the group runs past the tile: finish it from global memory
                uint32_t gj = i0 + NT; // first record of the next tile (known equal: s_eqn[NT-1])
                while (true) {
                    Rec nx = ld_rec(&m[gj]);
                    KeyRef ck = key_of_gid(p, nx.w);
                    bool better = true;
                    if (!p.mode_flush) {
                        uint64_t clo, chi;
                        ld_ts(ck.entry, ck.full_size, &clo, &chi);
                        better = !ts_greater(wlo, whi, clo, chi);
                        if (better) { wlo = clo; whi = chi; }
                    }
                    if (better) { ks = ck.klen + 8; fs = ck.full_size; src = (unsigned long long)(uintptr_t)ck.entry; wgid = nx.w; }
                    gj++;
                    if (gj >= lim_hi) break;
                    if (!key_equal(p, skip, nx, ld_rec(&m[gj]))) break;
                }
            }
        }
        bool tomb = fs == ks + 24;
        keep = (keep_tombstones || p.mode_flush || !tomb) ? 1u : 0u;
        // Bloom::set for every entry that is written (lsm_tree.rs:1049-1051), from the hashes k_extract left behind
        if (kHashRec && keep && p.hash_rec != nullptr && p.bloom.words != nullptr) {
            const uint4 hv = __ldg(&p.hash_rec[wgid]);
            uint32_t *words = p.bloom.words;
            bloom_probe_all((uint64_t)hv.x | ((uint64_t)hv.y << 32), (uint64_t)hv.z | ((uint64_t)hv.w << 32), p.bloom.k_num, p.bloom.bits,
                            p.bloom.bits_magic, [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
        }
    }
    if (!kFused) {
        if (i < span) res[i] = make_uint4((uint32_t)src, (uint32_t)(src >> 32), ks, keep ? fs : 0u); // holes: nothing emitted

        // tile aggregate (bytes, entries) for the offsets scan: three warp reductions (REDUX) -- the byte count in two 16-bit
        // halves, so that 32 entries of up to 4 GB each cannot overflow a 32-bit partial sum
        const uint32_t fk = keep ? fs : 0u;
        const uint32_t s_lo = __reduce_add_sync(0xFFFFFFFFu, fk & 0xFFFFu), s_hi = __reduce_add_sync(0xFFFFFFFFu, fk >> 16);
        unsigned long long vb = (unsigned long long)s_lo + ((unsigned long long)s_hi << 16);
        uint32_t vc = __reduce_add_sync(0xFFFFFFFFu, keep);
        __syncthreads(); // s_tlo / s_ks are dead: reuse them as the cross-warp scratch
        if ((tid & 31) == 0) { s_tlo[tid >> 5] = vb; s_ks[tid >> 5] = vc; }
        __syncthreads();
        if (tid == 0) {
            unsigned long long tb = 0;
            uint32_t tc = 0;
            for (int w = 0; w < NT / 32; w++) { tb += s_tlo[w]; tc += s_ks[w]; }
            p.tile_bytes[blockIdx.x] = tb;
            p.tile_count[blockIdx.x] = tc;
        }
        return;
    }

    // ---- fused: in-tile inclusive scan, chained scan over the tiles, then the writes k_emit would do
    const uint32_t lane = tid & 31, warp = tid >> 5;
    unsigned long long ib = keep ? fs : 0ull;
    uint32_t ic = keep;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long xb = __shfl_up_sync(0xFFFFFFFFu, ib, o);
        const uint32_t xc = __shfl_up_sync(0xFFFFFFFFu, ic, o);
        if (lane >= (uint32_t)o) { ib += xb; ic += xc; }
    }
    __syncthreads(); // s_tlo / s_ks / s_thi are dead: cross-warp scratch
    if (lane == 31) { s_tlo[warp] = ib; s_ks[warp] = ic; }
    __syncthreads();
    unsigned long long tb = 0, wb = 0;
    uint32_t tc = 0, wc = 0;
    for (int w = 0; w < NT / 32; w++) {
        if ((uint32_t)w < warp) { wb += s_tlo[w]; wc += s_ks[w]; }
        tb += s_tlo[w];
        tc += s_ks[w];
    }
    if (warp == 0) {
        unsigned long long *mine = p.scan_state + 2ull * tile_id;
        unsigned long long eb = 0;
        uint32_t ec = 0;
        if (tile_id == 0) {
            if (lane == 0) {
                st_volatile_u64(mine, (kScanPrefix << 62) | tb);
                __threadfence();
                st_volatile_u64(mine + 1, (kScanPrefix << 32) | tc);
            }
        } else {
            if (lane == 0) { // bytes word first, entries word second: a reader that sees the second sees the first
                st_volatile_u64(mine, (kScanAgg << 62) | tb);
                __threadfence();
                st_volatile_u64(mine + 1, (kScanAgg << 32) | tc);
            }
            int t = (int)tile_id - 1;
            while (true) {
                const int idx = t - (int)lane;
                unsigned long long vb2 = 0, vc2 = 0, stat = kScanPrefix;
                if (idx >= 0) {
                    const unsigned long long *q = p.scan_state + 2ull * (uint32_t)idx;
                    while (true) { // entries word, then bytes word; both must be at the same stage
                        vc2 = ld_volatile_u64(q + 1);
                        __threadfence();
                        vb2 = ld_volatile_u64(q);
                        if ((vc2 >> 32) != 0 && (vc2 >> 32) == (vb2 >> 62)) break;
                    }
                    stat = vc2 >> 32;
                }
                // lanes below the nearest tile that already holds an inclusive prefix add their aggregates, that tile its prefix
                const uint32_t pm = __ballot_sync(0xFFFFFFFFu, stat == kScanPrefix);
                const uint32_t first = (uint32_t)__ffs((int)pm) - 1; // pm != 0: lanes with idx < 0 report "prefix" (of nothing)
                unsigned long long cb = (lane <= first && idx >= 0) ? (vb2 & ((1ull << 62) - 1)) : 0ull;
                uint32_t cc = (lane <= first && idx >= 0) ? (uint32_t)vc2 : 0u;
#pragma unroll
                for (int o = 16; o; o >>= 1) {
                    cb += __shfl_xor_sync(0xFFFFFFFFu, cb, o);
                    cc += __shfl_xor_sync(0xFFFFFFFFu, cc, o);
                }
                eb += cb;
                ec += cc;
                if (pm) break;
                t -= 32;
            }
            if (lane == 0) {
                st_volatile_u64(mine, (kScanPrefix << 62) | (eb + tb));
                __threadfence();
                st_volatile_u64(mine + 1, (kScanPrefix << 32) | (unsigned long long)(ec + tc));
            }
        }
        if (lane == 0) {
            s_thi[0] = eb;
            s_fs[0] = ec;
            if ((unsigned long long)(tile_id + 1) * NT >= span) { // the last tile holds the totals
                Ctl *cw = p.ctl;
                cw->out_data_len = eb + tb;
                cw->out_items = ec + tc;
            }
        }
    }
    __syncthreads();
    if (!keep) return;
    const unsigned long long off = s_thi[0] + wb + ib - fs; // within this job's .data
    const uint32_t pos = s_fs[0] + wc + ic - 1;
    const unsigned long long file_off = off + p.out_offset_base;
    p.out_index[pos] = make_uint4((uint32_t)file_off, (uint32_t)(file_off >> 32), ks, fs);
    p.src_ptr[pos] = src;
    constexpr unsigned long long gt = kGatherTileBytes;
    for (unsigned long long bq = (off + gt - 1) / gt; bq * gt < off + fs && bq < p.tile_first_n; bq++) p.tile_first[bq] = pos;
}

// ------------------------------------------------------------------------------------
// K4b: offsets.  The survivor at merged position i becomes output entry `count before i`, at
// .data offset `bytes before i` (entry_writer.rs:81-86: offset = running sum of full_size).
// No inter-CTA waiting: (1) the per-tile aggregates are scanned in chunks of 1024 tiles, (2) one
// CTA scans the chunk totals, (3) every tile rescans its 256 records locally and emits
// out_index (the output .index file itself), src_ptr, and -- for every 16 KB tile of the
// output .data stream -- the entry that holds the tile's first byte (tile_first).

// block-wide exclusive scan of (bytes, count) over 1024 threads; returns the block totals
__device__ __forceinline__ void block_excl_scan_1024(unsigned long long &vb, uint32_t &vc, unsigned long long *s_b,
                                                     uint32_t *s_c, unsigned long long *tot_b, uint32_t *tot_c) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned long long ib = vb;
    uint32_t ic = vc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        unsigned long long xb = __shfl_up_sync(0xFFFFFFFFu, ib, o);
        uint32_t xc = __shfl_up_sync(0xFFFFFFFFu, ic, o);
        if (lane >= (uint32_t)o) { ib += xb; ic += xc; }
    }
    if (lane == 31) { s_b[warp] = ib; s_c[warp] = ic; }
    __syncthreads();
    if (warp == 0) {
        unsigned long long wb = s_b[lane];
        uint32_t wc = s_c[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned long long xb = __shfl_up_sync(0xFFFFFFFFu, wb, o);
            uint32_t xc = __shfl_up_sync(0xFFFFFFFFu, wc, o);
            if (lane >= (uint32_t)o) { wb += xb; wc += xc; }
        }
        s_b[lane] = wb;
        s_c[lane] = wc;
    }
    __syncthreads();
    *tot_b = s_b[31];
    *tot_c = s_c[31];
    vb = (warp ? s_b[warp - 1] : 0ull) + (ib - vb);
    vc = (warp ? s_c[warp - 1] : 0u) + (ic - vc);
}

// step 1: chunks of 1024 tiles, one CTA each: in-place exclusive scan + the chunk's totals
__global__ void __launch_bounds__(1024) k_scan_tiles(Params p) {
    pdl_trigger();
    pdl_wait();
    __shared__ unsigned long long s_b[32];
    __shared__ uint32_t s_c[32];
    const uint32_t n_tiles = (p.ctl->span + kResolveThreads - 1) / kResolveThreads;
    const uint32_t t = blockIdx.x * 1024u + threadIdx.x;
    if (blockIdx.x * 1024u >= n_tiles) return;
    unsigned long long vb = t < n_tiles ? p.tile_bytes[t] : 0ull;
    uint32_t vc = t < n_tiles ? p.tile_count[t] : 0u;
    unsigned long long tb;
    uint32_t tc;
    block_excl_scan_1024(vb, vc, s_b, s_c, &tb, &tc);
    if (t < n_tiles) { p.tile_bytes[t] = vb; p.tile_count[t] = vc; }
    if (threadIdx.x == 0) { p.chunk_bytes[blockIdx.x] = tb; p.chunk_count[blockIdx.x] = tc; }
}

// step 2: one CTA scans the chunk totals (1024x fewer than tiles) and publishes the job totals
__global__ void __launch_bounds__(1024) k_scan_chunks(Params p) {
    pdl_trigger();
    pdl_wait();
    __shared__ unsigned long long s_b[32];
    __shared__ uint32_t s_c[32];
    Ctl *c = p.ctl;
    const uint32_t n_tiles = (c->span + kResolveThreads - 1) / kResolveThreads;
    const uint32_t n_chunks = (n_tiles + 1023) / 1024;
    const uint32_t per = (n_chunks + 1023) / 1024;
    const uint32_t c0 = threadIdx.x * per < n_chunks ? threadIdx.x * per : n_chunks;
    const uint32_t c1 = c0 + per < n_chunks ? c0 + per : n_chunks;
    unsigned long long vb = 0;
    uint32_t vc = 0;
    for (uint32_t k = c0; k < c1; k++) { vb += p.chunk_bytes[k]; vc += p.chunk_count[k]; }
    unsigned long long tb;
    uint32_t tc;
    block_excl_scan_1024(vb, vc, s_b, s_c, &tb, &tc);
    for (uint32_t k = c0; k < c1; k++) {
        const unsigned long long b = p.chunk_bytes[k];
        const uint32_t n = p.chunk_count[k];
        p.chunk_bytes[k] = vb;
        p.chunk_count[k] = vc;
        vb += b;
        vc += n;
    }
    if (threadIdx.x == 0) { c->out_data_len = tb; c->out_items = tc; }
}

__global__ void __launch_bounds__(kResolveThreads) k_emit(Params p, const uint4 *res) {
    pdl_trigger();
    pdl_wait();
    constexpr int NT = kResolveThreads;
    __shared__ unsigned long long s_wb[NT / 32];
    __shared__ uint32_t s_wc[NT / 32];
    const uint32_t total = p.ctl->span;
    const uint32_t i0 = blockIdx.x * NT;
    if (i0 >= total) return;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t i = i0 + tid;
    uint4 it = make_uint4(0, 0, 0, 0);
    if (i < total) it = __ldg(&res[i]);
    const uint32_t fs = it.w;
    unsigned long long ib = fs;
    uint32_t ic = fs ? 1u : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        unsigned long long xb = __shfl_up_sync(0xFFFFFFFFu, ib, o);
        uint32_t xc = __shfl_up_sync(0xFFFFFFFFu, ic, o);
        if (lane >= (uint32_t)o) { ib += xb; ic += xc; }
    }
    if (lane == 31) { s_wb[warp] = ib; s_wc[warp] = ic; }
    __syncthreads();
    if (!fs) return;
    unsigned long long off = p.chunk_bytes[blockIdx.x >> 10] + p.tile_bytes[blockIdx.x] + ib - fs; // within this job's .data
    uint32_t pos = p.chunk_count[blockIdx.x >> 10] + p.tile_count[blockIdx.x] + ic - 1;
    for (uint32_t w = 0; w < warp; w++) { off += s_wb[w]; pos += s_wc[w]; }
    const unsigned long long src = (unsigned long long)it.x | ((unsigned long long)it.y << 32);
    const unsigned long long file_off = off + p.out_offset_base; // a key-range partition continues the file of the previous ones
    p.out_index[pos] = make_uint4((uint32_t)file_off, (uint32_t)(file_off >> 32), it.z, fs);
    p.src_ptr[pos] = src;
    // every gather tile whose first byte lies in [off, off + fs) starts inside this entry
    constexpr unsigned long long tb = kGatherTileBytes;
    unsigned long long b = (off + tb - 1) / tb;
    for (; b * tb < off + fs && b < p.tile_first_n; b++) p.tile_first[b] = pos;
}

// Flush-many epilogue.  The memtables' SSTables sit back to back in one output stream; every memtable's .index
// must carry offsets relative to its own .data file (entry_writer.rs:81-86 starts each file at 0).
// k_flush_table: what had been emitted before each memtable's first record (+ a sentinel row = the totals).
// k_rebase_index: subtract that from the memtable's index records.

__global__ void k_flush_table(Params p, const uint4 *res) {
    pdl_trigger();
    pdl_wait();
    const uint32_t mt = blockIdx.x * blockDim.x + threadIdx.x;
    if (mt > p.n_groups) return;
    const Ctl *c = p.ctl;
    unsigned long long bytes;
    unsigned long long items;
    if (mt == p.n_groups) {
        bytes = c->out_data_len;
        items = c->out_items;
    } else {
        const uint32_t pos = p.seg[p.n_levels][mt].start; // first merged position of the group
        if (pos >= c->span) {
            bytes = c->out_data_len;
            items = c->out_items;
        } else {
            const uint32_t tile = pos / kResolveThreads;
            bytes = p.chunk_bytes[tile >> 10] + p.tile_bytes[tile];
            items = (unsigned long long)p.chunk_count[tile >> 10] + p.tile_count[tile];
            for (uint32_t i = tile * kResolveThreads; i < pos; i++) {
                const uint32_t fs = res[i].w;
                bytes += fs;
                items += fs ? 1u : 0u;
            }
        }
    }
    p.mem_table[2 * mt] = bytes;
    p.mem_table[2 * mt + 1] = items;
}

__global__ void __launch_bounds__(256) k_rebase_index(Params p) {
    pdl_trigger();
    pdl_wait();
    const uint32_t e = blockIdx.x * 256u + threadIdx.x;
    if (e >= p.ctl->out_items) return;
    uint32_t lo = 0, hi = p.n_groups; // last group whose first entry is <= e (empty groups share a boundary)
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (p.mem_table[2 * mid + 1] <= e) lo = mid; else hi = mid;
    }
    uint4 rec = p.out_index[e];
    const unsigned long long off = ((unsigned long long)rec.x | ((unsigned long long)rec.y << 32)) - p.mem_table[2 * lo];
    rec.x = (uint32_t)off;
    rec.y = (uint32_t)(off >> 32);
    p.out_index[e] = rec;
}

// ------------------------------------------------------------------------------------
// K5: gather + bloom -- the roofline kernel.  Every surviving entry's bytes are read once
// from its input run and written once at its output offset.
//
// The output .data stream is cut into 16 KB tiles (1024 aligned 16-byte vectors), one CTA each.
//   * a vector that lies inside one entry = two aligned 16-byte source loads + a byte funnel
//     shift (source and destination are misaligned by an arbitrary byte count);
//   * a vector that straddles an entry boundary (one per entry) is built by a second, dense
//     pass: tail of entry j blended with the shifted head of entry j+1.
// No byte stores (bar the last <16 bytes of the stream), no overlap between CTAs: every output
// vector has exactly one writer.
// Bloom (fused epilogue): after its stores are issued the CTA hashes the key of every entry
// whose first byte lies in its tile (2 x SipHash-1-3 in one walk, one thread per entry) and
// sets k bits with atomicOr -- the filter (<= ~10 MB at the benchmark shapes) stays
// L2-resident and the key bytes are lines the copy has just touched.

__device__ __forceinline__ uint4 realign16_sel(uint4 A, uint4 B, uint32_t sh) {
    // branch-free version of realign16 for a per-lane shift
    const uint32_t bits = (sh & 3) * 8;
    const bool s2 = sh & 8, s1 = sh & 4;
    uint32_t c0 = s2 ? A.z : A.x, c1 = s2 ? A.w : A.y, c2 = s2 ? B.x : A.z;
    uint32_t c3 = s2 ? B.y : A.w, c4 = s2 ? B.z : B.x, c5 = s2 ? B.w : B.y;
    uint32_t d0 = s1 ? c1 : c0, d1 = s1 ? c2 : c1, d2 = s1 ? c3 : c2, d3 = s1 ? c4 : c3, d4 = s1 ? c5 : c4;
    return make_uint4(__funnelshift_r(d0, d1, bits), __funnelshift_r(d1, d2, bits), __funnelshift_r(d2, d3, bits),
                      __funnelshift_r(d3, d4, bits));
}

// ------------------------------------------------------------------------------------
// One staging pass, ONE block barrier, dense (thread-per-entry) straddle and bloom passes; the copy
// itself is done warp by warp on 2 KB sub-tiles: a warp finds the entry under its first byte once
// and then walks the (sorted) entry ends 512 bytes at a time, each lane counting how many entries
// end at or before its own vector (one OR-reduction + popcount per chunk).

#ifndef DBEEL_GATHER_MINB
#define DBEEL_GATHER_MINB (1536 / DBEEL_GATHER_THREADS) // 12 CTAs of 128 threads: 40 registers
#endif
__global__ void __launch_bounds__(kGatherThreads, DBEEL_GATHER_MINB) k_gather(Params p) {
    pdl_trigger();
    pdl_wait();
    constexpr int NT = kGatherThreads;
    constexpr int VPT = kGatherVecsPerThread;
    __shared__ unsigned long long s_adj[kGatherMaxEntries]; // entry address minus its tile-relative start
    __shared__ int s_r0[kGatherMaxEntries], s_r1[kGatherMaxEntries];
    __shared__ uint32_t s_ks[kGatherMaxEntries];
    const Ctl *c = p.ctl;
    const unsigned long long out_len = c->out_data_len;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile_id = blockIdx.x;
    const unsigned long long T0 = (unsigned long long)tile_id * kGatherTileBytes;
    if (T0 >= out_len) return;
    const uint32_t tile_len = out_len - T0 < kGatherTileBytes ? (uint32_t)(out_len - T0) : (uint32_t)kGatherTileBytes;
    const uint32_t e_lo = p.tile_first[tile_id];
    const uint32_t e_hi = T0 + kGatherTileBytes < out_len ? p.tile_first[tile_id + 1] : c->out_items - 1;
    const uint32_t ne = e_hi - e_lo + 1; // <= kGatherMaxEntries: every entry is >= 32 bytes
    for (uint32_t j = tid; j < ne; j += NT) {
        const uint4 rec = p.out_index[e_lo + j];
        const unsigned long long d0 = ((unsigned long long)rec.x | ((unsigned long long)rec.y << 32)) - p.out_offset_base;
        const long long r0 = (long long)d0 - (long long)T0; // < 0 only for the tile's first entry
        const long long r1 = r0 + (long long)rec.w;
        s_adj[j] = p.src_ptr[e_lo + j] - (unsigned long long)r0;
        s_r0[j] = r0 < -0x7FFFFFFFll ? -0x7FFFFFFF : (int)r0;
        s_r1[j] = r1 > 0x7FFFFFFFll ? 0x7FFFFFFF : (int)r1;
        s_ks[j] = rec.z;
    }
    __syncthreads();

    // ---- copy: warp w owns bytes [w * 2 KB, (w + 1) * 2 KB) of the tile
    uint8_t *dst_tile = p.out_data + T0;
    const int sub0 = (int)(warp * (uint32_t)(32 * VPT * 16));
    if ((uint32_t)sub0 < tile_len) {
        // j = the entry that holds byte sub0 = number of entries ending at or before it (ends ascend).
        uint32_t j = 0;
        for (uint32_t base = 0; base + 1 < ne; base += 32) { // ballot-count 32 entries at a time; the last entry never counts
            const uint32_t i = base + lane;
            j += __popc(__ballot_sync(0xFFFFFFFFu, i + 1 < ne && s_r1[i] <= sub0));
        }
        uint4 A[VPT], B[VPT];
        uint32_t sh[VPT];
        bool pure[VPT];
        const uint32_t lanes_le = 0xFFFFFFFFu >> (31 - lane); // bits 0..lane
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            const int cb = sub0 + k * 512; // this 512-byte chunk: one vector per lane
            const int b0 = cb + (int)lane * 16;
            // Entries that end inside the chunk, i.e. in (cb, cb + 512]: at most 17 (entries are >= 32 bytes),
            // lane l looks at entry j + l.  An end at r1 precedes the vectors t = ceil((r1 - cb) / 16) .. 31,
            // and distinct entries have distinct t, so one OR-reduction builds the whole chunk's map.
            const uint32_t i = j + lane;
            const int r1 = i + 1 < ne ? s_r1[i] : 0x7FFFFFFF;
            const bool ends_here = r1 <= cb + 512;
            const uint32_t t = (uint32_t)((ends_here ? r1 : cb + 16) - cb + 15) >> 4; // 1..32 when ends_here
            const uint32_t ends = __reduce_or_sync(0xFFFFFFFFu, (ends_here && t < 32) ? (1u << t) : 0u);
            const uint32_t cnt = __popc(ends & lanes_le); // entries ending at or before my vector's first byte
            const uint32_t adv = __popc(__ballot_sync(0xFFFFFFFFu, ends_here));
            const uint32_t e = j + cnt; // entry that holds byte b0
            j += adv;                   // entry that holds the next chunk's first byte
            // Loads are unconditional (no divergent branch around them): a vector that is not wholly inside
            // entry e -- it straddles e's end, or lies past the end of the stream -- reads the last full vector
            // of e instead (always valid memory: entries are >= 32 bytes) and simply is not stored.
            const int r1e = s_r1[e];
            pure[k] = (uint32_t)b0 + 16 <= tile_len && b0 + 16 <= r1e;
            const int bl = b0 + 16 <= r1e ? b0 : r1e - 16;
            const uintptr_t sa = (uintptr_t)(s_adj[e] + (unsigned long long)(long long)bl);
            sh[k] = (uint32_t)(sa & 15);
            const uint4 *sv = reinterpret_cast<const uint4 *>(sa - sh[k]);
            A[k] = __ldg(sv);
            B[k] = __ldg(sh[k] ? sv + 1 : sv);
        }
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            const uint32_t v = (uint32_t)(sub0 >> 4) + (uint32_t)k * 32 + lane;
            if (pure[k]) reinterpret_cast<uint4 *>(dst_tile)[v] = realign16_sel(A[k], B[k], sh[k]);
        }
    }

    // ---- the vector that holds the last byte of entry j: tail of j blended with the head of j+1
    for (uint32_t j = tid; j < ne; j += NT) {
        const int r1 = s_r1[j];
        if (r1 <= 0 || (r1 & 15) == 0 || r1 > (int)tile_len) continue;
        const uint32_t v = (uint32_t)r1 >> 4;
        const uint32_t b0 = v * 16;
        const uint32_t t = (uint32_t)r1 - b0; // tail bytes of entry j in this vector: 1..15
        const uintptr_t sa = (uintptr_t)(s_adj[j] + b0);
        const uint32_t s0 = (uint32_t)(sa & 15);
        const uint4 *sv = reinterpret_cast<const uint4 *>(sa - s0);
        const uint4 TA = __ldg(sv);
        const uint4 TB = __ldg(s0 + t > 16 ? sv + 1 : sv);
        uint4 o = realign16_sel(TA, TB, s0);
        if (b0 + 16 <= tile_len) {
            const uintptr_t ha = (uintptr_t)(s_adj[j + 1] + (unsigned long long)(long long)s_r0[j + 1]); // first byte of entry j+1
            const uint32_t hs = (uint32_t)(ha & 15);
            const uint4 *hv = reinterpret_cast<const uint4 *>(ha - hs);
            const uint4 HA = __ldg(hv);
            const uint4 HB = __ldg(hs ? hv + 1 : hv);
            const uint4 H = realign16_sel(HA, HB, hs);
            const uint4 HU = realign16_sel(make_uint4(0, 0, 0, 0), H, 16 - t);
            const uint32_t wfull = t >> 2, bits = (t & 3) * 8;
            const uint32_t mmix = bits ? (0xFFFFFFFFu >> (32 - bits)) : 0u;
            uint32_t ow[4] = {o.x, o.y, o.z, o.w}, hw[4] = {HU.x, HU.y, HU.z, HU.w};
#pragma unroll
            for (uint32_t q = 0; q < 4; q++) {
                const uint32_t mk = q < wfull ? 0xFFFFFFFFu : (q == wfull ? mmix : 0u);
                ow[q] = (ow[q] & mk) | (hw[q] & ~mk);
            }
            reinterpret_cast<uint4 *>(dst_tile)[v] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        } else { // ragged end of the whole stream: never write past out_data_len
            const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
            for (uint32_t b = 0; b < t; b++) dst_tile[b0 + b] = (uint8_t)(ow[b >> 2] >> ((b & 3) * 8));
        }
    }

    // ---- bloom (fused epilogue): entries whose first byte lies in this tile
    if (p.bloom.words != nullptr && p.hash_rec == nullptr && !p.bloom_elsewhere) {
        for (uint32_t j = tid; j < ne; j += NT) {
            const int r0 = s_r0[j];
            if (r0 < 0 || r0 >= (int)kGatherTileBytes) continue;
            const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)(s_adj[j] + (unsigned long long)r0)) + 8;
            const uint64_t klen = s_ks[j] - 8;
            uint64_t h0, h1;
            sip13_pair_vec_u8(p.bloom.sip, klen, [key](uint64_t q) { return ld_u64_unaligned(key + 8 * q); }, &h0, &h1);
            uint32_t *words = p.bloom.words;
            bloom_probe_all(h0, h1, p.bloom.k_num, p.bloom.bits, p.bloom.bits_magic,
                            [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
        }
    }
}

// ------------------------------------------------------------------------------------
// K5, 32 bytes per lane (the default).  Same tiles, same staging, same one barrier as k_gather; what changes is the
// granule every lane moves: a 32-byte block = three aligned 16-byte loads + one 32-byte store (stg256) instead of
// 2 x (two loads + one 128-bit store).  Per output byte that halves the vector -> entry mapping (one OR-reduction +
// popcount now covers 1 KB) and the address arithmetic, and takes the load over-fetch from 2x to 1.5x.  A block that holds an entry boundary (one per entry at most: entries are >= 32 bytes) is
// left to a second, dense pass that writes its two 16-byte halves: tail of entry j, head of entry j + 1, or a blend.
// The bloom epilogue only runs when k_extract did not hash (p.hash_rec == null).

__device__ __forceinline__ void realign32(const uint4 A, const uint4 B, const uint4 C, uint32_t sh, uint32_t out[8]) {
    // 32 output bytes starting `sh` (0..15) bytes into the 48-byte window {A, B, C}; C is not read when sh == 0
    const uint32_t bits = (sh & 3) * 8;
    const bool s2 = sh & 8, s1 = sh & 4;
    const uint32_t w[12] = {A.x, A.y, A.z, A.w, B.x, B.y, B.z, B.w, C.x, C.y, C.z, C.w};
    uint32_t c[10], d[9];
#pragma unroll
    for (int i = 0; i < 10; i++) c[i] = s2 ? w[i + 2] : w[i];
#pragma unroll
    for (int i = 0; i < 9; i++) d[i] = s1 ? c[i + 1] : c[i];
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = __funnelshift_r(d[i], d[i + 1], bits);
}

// one 32-byte aligned block: sm_90 has no 256-bit global access, so it leaves as two 128-bit stores (STG.E.128)
__device__ __forceinline__ void stg256(void *dst, const uint32_t v[8]) {
    asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
    asm volatile("st.global.v4.b32 [%0+16], {%1, %2, %3, %4};" ::"l"(dst), "r"(v[4]), "r"(v[5]), "r"(v[6]), "r"(v[7]) : "memory");
}

// 16 bytes at an arbitrary address, `need` of them wanted: the second aligned load is skipped when the first one holds them all
__device__ __forceinline__ uint4 ld16_any(uintptr_t sa, uint32_t need) {
    const uint32_t s0 = (uint32_t)(sa & 15);
    const uint4 *sv = reinterpret_cast<const uint4 *>(sa - s0);
    const uint4 TA = __ldg(sv);
    const uint4 TB = __ldg(s0 + need > 16 ? sv + 1 : sv);
    return realign16_sel(TA, TB, s0);
}

__device__ __forceinline__ void ldg256_nc(const void *p, uint32_t v[8]) { // one 32-byte aligned chunk as two LDG.E.128
    asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(p));
    asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4+16];" : "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7]) : "l"(p));
}

// 32 bytes at an arbitrary address of which bytes [lo, hi) are wanted (0 <= lo < hi <= 32): only the aligned 32-byte chunks
// that hold wanted bytes are loaded (a lane that needs one chunk costs the L1 data pipe one wavefront, not two)
__device__ __forceinline__ void ld32_any(uintptr_t a, uint32_t lo, uint32_t hi, uint32_t out[8]) {
    const uint32_t s0 = (uint32_t)(a & 31);
    const uintptr_t base = a - s0;
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = 0u;
    if (lo < 32u - s0) ldg256_nc(reinterpret_cast<const void *>(base), w);          // chunk 0 = bytes [0, 32 - s0) of the block
    if (hi > 32u - s0) ldg256_nc(reinterpret_cast<const void *>(base + 32), w + 8); // chunk 1 = bytes [32 - s0, 32)
    window32(w, s0, out);
}

constexpr int kG32Vpt = (int)(kGatherTileBytes / (32ull * kGatherThreads)); // 1 KB chunks per warp
static_assert(kGatherTileBytes == 32ull * kGatherThreads * kG32Vpt, "gather tile = 32 bytes x lanes x chunks");

#ifndef DBEEL_GATHER32_MINB
#define DBEEL_GATHER32_MINB (1536 / DBEEL_GATHER_THREADS)
#endif
#ifndef DBEEL_GATHER32W_MINB
#define DBEEL_GATHER32W_MINB 9
#endif
// kBloomWarp: a fifth warp does nothing but the filter -- the tile's keys are hashed WHILE the four copy warps wait for their
// payload loads, instead of after their stores by the same threads (the fused epilogue is a ~600-instruction dependent chain
// per entry on 27 of 128 lanes: it lengthens every CTA's life by about a fifth).
// kRot: the two dense per-entry passes run on DIFFERENT warps -- entry j's boundary block is written by thread (j + 96) mod 128
// (warp 3 first), its key is hashed by thread (j + 32) mod 128 (warp 1 first).  A tile holds ~27 entries of 305 bytes, so with
// the plain j = tid mapping warp 0 alone walks copy -> boundary loads -> key loads -> 600 dependent hash instructions while
// warps 1-3 have exited but still hold their slots: the CTA lives as long as its slowest warp.
// kSplit: the filter is filled by CTAs OF THEIR OWN, interleaved with the copy CTAs in the same grid (every ~5th block): a
// filter CTA takes 128 consecutive output entries, one key per thread, all lanes busy, and runs on an SM next to copy CTAs
// that are waiting for their payload -- its ~600 dependent hash instructions per key fill issue slots the copy leaves idle
// instead of lengthening every copy CTA's life.  (Two kernels on two streams do not co-run when each fills the GPU; blocks
// of one grid do.)  The key bytes are the first granule of an entry the copy CTA of the same region touches within a few
// microseconds either way: an L2 hit for whichever comes second.  Block b is a filter block iff floor((b+1) nb / G) >
// floor(b nb / G) (nb filter blocks spread evenly over the G blocks of the grid); it is filter block floor(b nb / G), and
// a copy block is tile b - floor(b nb / G).
// kLean (the default since round 2, DBEEL_GATHER=10; 1 = the two-halves pass below): the entry-boundary blocks with fewer trips
// through the L1 data pipe, where every lane's access is a wavefront of its own (the one-lane-per-entry passes -- boundary
// blocks, key loads, the filter's REDs -- issue most of the kernel's wavefronts; the copy proper a minority).  The
// tail of entry j and the head of entry j + 1 each come from the aligned 32-byte chunks that hold wanted bytes (ldg256_nc,
// one or two per side), are blended in registers and leave in one 32-byte store instead of 6 loads + 2 stores.  The same idea
// applied to the key loads (two aligned 16-byte chunks per key, or two lanes per key with one SipHash each) was slower.
template <bool kBloomWarp, bool kRot, bool kSplit, bool kLean = false>
__global__ void __launch_bounds__(kGatherThreads + (kBloomWarp ? 32 : 0), kBloomWarp ? DBEEL_GATHER32W_MINB : DBEEL_GATHER32_MINB)
k_gather32(Params p) {
    pdl_trigger();
    pdl_wait();
    constexpr int NT = kGatherThreads;            // copy threads
    constexpr int NTA = NT + (kBloomWarp ? 32 : 0); // all threads
    uint32_t tile_of_block = blockIdx.x;
    if (kSplit) {
        const uint64_t nb = p.bloom_ctas, G = gridDim.x;
        const uint32_t q0 = (uint32_t)((uint64_t)blockIdx.x * nb / G), q1 = (uint32_t)(((uint64_t)blockIdx.x + 1) * nb / G);
        if (q1 != q0) { // filter block q0: output entries [128 q0, 128 q0 + 128)
            const uint32_t e = q0 * (uint32_t)NT + threadIdx.x;
            if (p.bloom.words == nullptr || e >= p.ctl->out_items) return;
            const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)__ldg(&p.src_ptr[e])) + 8;
            const uint64_t klen = __ldg(&p.out_index[e]).z - 8;
            uint64_t h0, h1;
            sip13_pair_vec_u8(p.bloom.sip, klen, [key](uint64_t q) { return ld_u64_unaligned(key + 8 * q); }, &h0, &h1);
            uint32_t *words = p.bloom.words;
            bloom_probe_all(h0, h1, p.bloom.k_num, p.bloom.bits, p.bloom.bits_magic,
                            [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
            return;
        }
        tile_of_block = blockIdx.x - q0;
    }
    __shared__ unsigned long long s_adj[kGatherMaxEntries]; // entry address minus its tile-relative start
    __shared__ int s_r0[kGatherMaxEntries], s_r1[kGatherMaxEntries];
    __shared__ uint32_t s_ks[kGatherMaxEntries];
    const Ctl *c = p.ctl;
    const unsigned long long out_len = c->out_data_len;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile_id = tile_of_block;
    const unsigned long long T0 = (unsigned long long)tile_id * kGatherTileBytes;
    if (T0 >= out_len) return;
    const uint32_t tile_len = out_len - T0 < kGatherTileBytes ? (uint32_t)(out_len - T0) : (uint32_t)kGatherTileBytes;
    const uint32_t e_lo = p.tile_first[tile_id];
    const uint32_t e_hi = T0 + kGatherTileBytes < out_len ? p.tile_first[tile_id + 1] : c->out_items - 1;
    const uint32_t ne = e_hi - e_lo + 1; // <= kGatherMaxEntries: every entry is >= 32 bytes
    const bool hash_here = !kSplit && p.bloom.words != nullptr && p.hash_rec == nullptr && !p.bloom_elsewhere;
    for (uint32_t j = tid; j < ne; j += NTA) {
        const uint4 rec = p.out_index[e_lo + j];
        const unsigned long long d0 = ((unsigned long long)rec.x | ((unsigned long long)rec.y << 32)) - p.out_offset_base;
        const long long r0 = (long long)d0 - (long long)T0; // < 0 only for the tile's first entry
        const long long r1 = r0 + (long long)rec.w;
        s_adj[j] = p.src_ptr[e_lo + j] - (unsigned long long)r0;
        s_r0[j] = r0 < -0x7FFFFFFFll ? -0x7FFFFFFF : (int)r0;
        s_r1[j] = r1 > 0x7FFFFFFFll ? 0x7FFFFFFF : (int)r1;
        if (hash_here) s_ks[j] = rec.z;
    }
    __syncthreads();

    if (kBloomWarp && warp == NT / 32) { // the filter warp: entries whose first byte lies in this tile
        if (hash_here) {
            for (uint32_t j = lane; j < ne; j += 32) {
                const int r0 = s_r0[j];
                if (r0 < 0 || r0 >= (int)kGatherTileBytes) continue;
                const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)(s_adj[j] + (unsigned long long)r0)) + 8;
                const uint64_t klen = s_ks[j] - 8;
                uint64_t h0, h1;
                sip13_pair_vec_u8(p.bloom.sip, klen, [key](uint64_t q) { return ld_u64_unaligned(key + 8 * q); }, &h0, &h1);
                uint32_t *words = p.bloom.words;
                bloom_probe_all(h0, h1, p.bloom.k_num, p.bloom.bits, p.bloom.bits_magic,
                                [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
            }
        }
        return;
    }

    // ---- copy: warp w owns bytes [w * 2 KB, (w + 1) * 2 KB) of the tile, 1 KB (32 lanes x 32 bytes) at a time
    uint8_t *dst_tile = p.out_data + T0;
    const int sub0 = (int)(warp * (uint32_t)(kG32Vpt * 1024));
    if ((uint32_t)sub0 < tile_len) {
        uint32_t j = 0; // the entry that holds byte sub0 = number of entries ending at or before it (ends ascend)
        for (uint32_t base = 0; base + 1 < ne; base += 32) {
            const uint32_t i = base + lane;
            j += __popc(__ballot_sync(0xFFFFFFFFu, i + 1 < ne && s_r1[i] <= sub0));
        }
        uint4 A[kG32Vpt], B[kG32Vpt], C[kG32Vpt];
        uint32_t sh[kG32Vpt];
        bool pure[kG32Vpt];
        const uint32_t lanes_le = 0xFFFFFFFFu >> (31 - lane); // bits 0..lane
#pragma unroll
        for (int k = 0; k < kG32Vpt; k++) {
            const int cb = sub0 + k * 1024;
            const int b0 = cb + (int)lane * 32;
            // Entries that end inside the chunk, i.e. in (cb, cb + 1024]: at most 32, lane l looks at entry j + l.  An end at
            // r1 precedes the blocks t = ceil((r1 - cb) / 32) .. 31; distinct entries have distinct t.
            const uint32_t i = j + lane;
            const int r1 = i + 1 < ne ? s_r1[i] : 0x7FFFFFFF;
            const bool ends_here = r1 <= cb + 1024;
            const uint32_t t = (uint32_t)((ends_here ? r1 : cb + 32) - cb + 31) >> 5; // 1..32 when ends_here
            const uint32_t ends = __reduce_or_sync(0xFFFFFFFFu, (ends_here && t < 32) ? (1u << t) : 0u);
            const uint32_t cnt = __popc(ends & lanes_le); // entries ending at or before my block's first byte
            const uint32_t adv = __popc(__ballot_sync(0xFFFFFFFFu, ends_here));
            const uint32_t e = j + cnt; // entry that holds byte b0
            j += adv;                   // entry that holds the next chunk's first byte
            // Unconditional loads: a block that is not wholly inside entry e (it holds e's end, or lies past the end of the
            // stream) reads the last 32 bytes of e instead (always valid: entries are >= 32 bytes) and is not stored here.
            const int r1e = s_r1[e];
            pure[k] = (uint32_t)b0 + 32 <= tile_len && b0 + 32 <= r1e;
            const int bl = b0 + 32 <= r1e ? b0 : r1e - 32;
            const uintptr_t sa = (uintptr_t)(s_adj[e] + (unsigned long long)(long long)bl);
            sh[k] = (uint32_t)(sa & 15);
            const uint4 *sv = reinterpret_cast<const uint4 *>(sa - sh[k]);
            A[k] = __ldg(sv); // (skipping these loads for the ~27 blocks per tile that are not stored here was slower)
            B[k] = __ldg(sv + 1);
            C[k] = __ldg(sh[k] ? sv + 2 : sv + 1);
        }
#pragma unroll
        for (int k = 0; k < kG32Vpt; k++) {
            if (pure[k]) {
                uint32_t o[8];
                realign32(A[k], B[k], C[k], sh[k], o);
                stg256(dst_tile + sub0 + k * 1024 + (int)lane * 32, o);
            }
        }
    }

    // ---- the 32-byte block that holds the last byte of entry j (unless j ends on a block boundary)
    if (kLean) {
        for (uint32_t j = tid; j < ne; j += NT) {
            const int r1 = s_r1[j];
            if (r1 <= 0 || (r1 & 31) == 0 || r1 > (int)tile_len) continue;
            const uint32_t b0 = (uint32_t)r1 & ~31u, t = (uint32_t)r1 - b0; // t = 1..31 bytes of entry j in this block
            uint32_t T[8];
            ld32_any((uintptr_t)(s_adj[j] + b0), 0u, t, T);
            if (b0 + 32u <= tile_len) { // the rest of the block is the head of entry j + 1 (entries are >= 32 bytes)
                uint32_t H[8], O[8];
                ld32_any((uintptr_t)(s_adj[j + 1] + b0), t, 32u, H);
                blend32(T, H, t, O);
                stg256(dst_tile + b0, O);
            } else { // ragged end of the whole stream: never write past out_data_len
                uint32_t tw[8];
#pragma unroll
                for (int q = 0; q < 8; q++) tw[q] = T[q];
                for (uint32_t b = 0; b < t; b++) dst_tile[b0 + b] = (uint8_t)(tw[b >> 2] >> ((b & 3) * 8));
            }
        }
    }
    for (uint32_t j = kLean ? ne : (kRot ? (tid + NT - 96u) % NT : tid); j < ne; j += NT) {
        const int r1 = s_r1[j];
        if (r1 <= 0 || (r1 & 31) == 0 || r1 > (int)tile_len) continue;
        const bool has_next = j + 1 < ne;
#pragma unroll
        for (int half = 0; half < 2; half++) {
            const uint32_t b0 = ((uint32_t)r1 & ~31u) + 16u * half;
            if (b0 >= tile_len) continue;     // past the end of the stream
            const int t = r1 - (int)b0;       // bytes of entry j in this vector: <= 0 none, >= 16 all
            uint4 o;
            if (t >= 16) {
                o = ld16_any((uintptr_t)(s_adj[j] + b0), 16);
            } else if (t <= 0) {
                if (!has_next) continue;
                o = ld16_any((uintptr_t)(s_adj[j + 1] + b0), 16);
            } else {
                o = ld16_any((uintptr_t)(s_adj[j] + b0), (uint32_t)t);
                if (b0 + 16 <= tile_len) { // blend with the head of entry j + 1
                    const uint4 H = ld16_any((uintptr_t)(s_adj[j + 1] + (unsigned long long)(long long)r1), 16);
                    const uint4 HU = realign16_sel(make_uint4(0, 0, 0, 0), H, 16 - (uint32_t)t);
                    const uint32_t wfull = (uint32_t)t >> 2, bits = ((uint32_t)t & 3) * 8;
                    const uint32_t mmix = bits ? (0xFFFFFFFFu >> (32 - bits)) : 0u;
                    uint32_t ow[4] = {o.x, o.y, o.z, o.w}, hw[4] = {HU.x, HU.y, HU.z, HU.w};
#pragma unroll
                    for (uint32_t q = 0; q < 4; q++) {
                        const uint32_t mk = q < wfull ? 0xFFFFFFFFu : (q == wfull ? mmix : 0u);
                        ow[q] = (ow[q] & mk) | (hw[q] & ~mk);
                    }
                    o = make_uint4(ow[0], ow[1], ow[2], ow[3]);
                } else { // ragged end of the whole stream: never write past out_data_len
                    const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
                    for (int b = 0; b < t; b++) dst_tile[b0 + b] = (uint8_t)(ow[b >> 2] >> ((b & 3) * 8));
                    continue;
                }
            }
            reinterpret_cast<uint4 *>(dst_tile)[b0 >> 4] = o;
        }
    }

    // ---- bloom (fused epilogue), only when k_extract did not hash: entries whose first byte lies in this tile
    if (!kBloomWarp && hash_here) {
        for (uint32_t j = kRot ? (tid + NT - 32u) % NT : tid; j < ne; j += NT) {
            const int r0 = s_r0[j];
            if (r0 < 0 || r0 >= (int)kGatherTileBytes) continue;
            const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)(s_adj[j] + (unsigned long long)r0)) + 8;
            const uint64_t klen = s_ks[j] - 8;
            uint64_t h0, h1;
            sip13_pair_vec_u8(p.bloom.sip, klen, [key](uint64_t q) { return ld_u64_unaligned(key + 8 * q); }, &h0, &h1);
            uint32_t *words = p.bloom.words;
            bloom_probe_all(h0, h1, p.bloom.k_num, p.bloom.bits, p.bloom.bits_magic,
                            [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
        }
    }
}

// ------------------------------------------------------------------------------------
// K5, TMA-staged (the default): "SSTable data blocks staged from HBM into shared memory via TMA".
//
// Why: k_gather / k_gather32 are neither DRAM- nor issue-bound.  A CTA walks its phases one
// after the other -- tile_first -> out_index / src_ptr -> payload loads -> stores -> boundary loads -> key loads -- and
// every arrow is a memory round trip that only the OTHER resident CTAs can cover.  Here the payload of a tile comes in
// through the bulk-copy engine instead: one cp.async.bulk per entry (its 16-byte-aligned superset, <= tile bytes + 30),
// all completing on one mbarrier, issued a whole tile AHEAD (two shared-memory stages), with the metadata of the tile
// after that already travelling in registers.  By the time a tile is processed its bytes are in shared memory; the byte
// realignment (the bulk engine preserves address mod 16, source and destination offsets differ by an arbitrary byte
// count) runs from shared memory with LDS.128 + funnel shifts, the output leaves in 32-byte blocks (stg256), and the bloom hashes
// read their keys from shared memory too.  Persistent CTAs, one tile per iteration.
//
//   iteration q:   metadata of tile q+1 (registers) -> shared memory, prefix sum of the staged lengths, bulk copies issued
//                  global loads for the metadata of tile q+2 and the tile_first pair of tile q+3 (consumed next iteration)
//                  wait for tile q's mbarrier -> copy / boundary blocks / bloom from stage q & 1
//
// Staging layout of a tile: entry j's in-tile part [r0c, r1c) is copied from src_lo = src & ~15 as len = ceil16(sh + n) bytes
// to stage offset base_j = sum of the earlier lengths, so its byte at tile position b lives at sadj_j + b with
// sadj_j = base_j + sh - r0c.

constexpr int kGtThreads = kGatherThreads;
constexpr int kGtPer = (kGatherMaxEntries + kGtThreads - 1) / kGtThreads;          // entries a thread may have to stage
constexpr uint32_t kGtStageBytes = (uint32_t)kGatherTileBytes + 32u * kGatherMaxEntries + 128u; // payload + per-entry slack
#ifndef DBEEL_GT_CTAS
#define DBEEL_GT_CTAS 4
#endif

struct GtMeta {
    unsigned long long adj[kGatherMaxEntries]; // global address of the entry minus its tile-relative start
    uint32_t sadj[kGatherMaxEntries];          // stage offset of the entry's byte at tile position 0
    int r0[kGatherMaxEntries], r1[kGatherMaxEntries];
    uint32_t ks[kGatherMaxEntries];
    uint32_t ne, tile_len;
    unsigned long long T0;
};
constexpr uint32_t kGtSmem = 2u * kGtStageBytes + 2u * (uint32_t)sizeof(GtMeta) + 64u;

__device__ __forceinline__ uint4 lds16_any(const uint8_t *stage, uint32_t off, uint32_t need) {
    const uint32_t s0 = off & 15u;
    const uint4 *sv = reinterpret_cast<const uint4 *>(stage + (off - s0));
    const uint4 TA = *sv;
    const uint4 TB = *(s0 + need > 16 ? sv + 1 : sv);
    return realign16_sel(TA, TB, s0);
}

__global__ void __launch_bounds__(kGtThreads, DBEEL_GT_CTAS) k_gather_tma(Params p) {
    pdl_trigger();
    pdl_wait();
    constexpr int NT = kGtThreads;
    extern __shared__ __align__(128) uint8_t gt_raw[];
    auto stage_ptr = [&](uint32_t st) -> uint8_t * { return gt_raw + st * kGtStageBytes; };
    auto meta_ptr = [&](uint32_t st) -> GtMeta * { return reinterpret_cast<GtMeta *>(gt_raw + 2 * kGtStageBytes) + st; };
    __shared__ __align__(8) uint64_t s_bar[2];
    __shared__ uint32_t s_scan[NT / 32];
    const Ctl *c = p.ctl;
    const unsigned long long out_len = c->out_data_len;
    const uint32_t out_items = c->out_items;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t n_tiles = (uint32_t)((out_len + kGatherTileBytes - 1) / kGatherTileBytes);
    const uint32_t G = gridDim.x;
    if (blockIdx.x >= n_tiles) return;
    if (tid == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // ---- the three pipeline steps that run ahead of the tile being copied
    struct TF { uint32_t e_lo, ne; };
    auto load_tf = [&](uint32_t t) -> TF { // which entries overlap tile t
        TF r;
        r.e_lo = 0; r.ne = 0;
        if (t < n_tiles) {
            r.e_lo = __ldg(&p.tile_first[t]);
            const uint32_t e_hi = t + 1 < n_tiles ? __ldg(&p.tile_first[t + 1]) : out_items - 1;
            r.ne = e_hi - r.e_lo + 1;
        }
        return r;
    };
    auto load_recs = [&](const TF &tf, uint4 rec[kGtPer], unsigned long long src[kGtPer]) { // their index records / addresses
#pragma unroll
        for (int k = 0; k < kGtPer; k++) {
            const uint32_t j = tid + (uint32_t)k * NT;
            rec[k] = make_uint4(0, 0, 0, 0);
            src[k] = 0;
            if (j < tf.ne) {
                rec[k] = __ldg(&p.out_index[tf.e_lo + j]);
                src[k] = __ldg(&p.src_ptr[tf.e_lo + j]);
            }
        }
    };
    auto publish = [&](uint32_t st, uint32_t t, const TF &tf, const uint4 rec[kGtPer], const unsigned long long src[kGtPer]) {
        GtMeta &m = *meta_ptr(st);
        const unsigned long long T0 = (unsigned long long)t * kGatherTileBytes;
        const uint32_t tile_len = out_len - T0 < kGatherTileBytes ? (uint32_t)(out_len - T0) : (uint32_t)kGatherTileBytes;
        uint32_t carry = 0;
#pragma unroll
        for (int k = 0; k < kGtPer; k++) {
            if ((uint32_t)k * NT >= tf.ne) break; // uniform
            const uint32_t j = tid + (uint32_t)k * NT;
            uint32_t len = 0, sh = 0;
            int r0c = 0;
            unsigned long long src_lo = 0;
            if (j < tf.ne) {
                const unsigned long long d0 = ((unsigned long long)rec[k].x | ((unsigned long long)rec[k].y << 32)) - p.out_offset_base;
                const long long r0 = (long long)d0 - (long long)T0; // < 0 only for the tile's first entry
                const long long r1 = r0 + (long long)rec[k].w;
                const unsigned long long adj = src[k] - (unsigned long long)r0;
                m.adj[j] = adj;
                m.r0[j] = r0 < -0x7FFFFFFFll ? -0x7FFFFFFF : (int)r0;
                m.r1[j] = r1 > 0x7FFFFFFFll ? 0x7FFFFFFF : (int)r1;
                m.ks[j] = rec[k].z;
                r0c = r0 < 0 ? 0 : (int)r0;
                const int r1c = r1 > (long long)tile_len ? (int)tile_len : (int)r1;
                const unsigned long long src_c = adj + (unsigned long long)r0c;
                sh = (uint32_t)(src_c & 15);
                src_lo = src_c - sh;
                len = (sh + (uint32_t)(r1c - r0c) + 15u) & ~15u;
            }
            // exclusive prefix of len over the 128 entries of this round, in entry order
            uint32_t inc = len;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, inc, o);
                if (lane >= (uint32_t)o) inc += x;
            }
            __syncthreads(); // s_scan of the previous round / call has been read
            if (lane == 31) s_scan[warp] = inc;
            __syncthreads();
            uint32_t before = carry, total = 0;
#pragma unroll
            for (int w = 0; w < NT / 32; w++) {
                if ((uint32_t)w < warp) before += s_scan[w];
                total += s_scan[w];
            }
            const uint32_t base = before + inc - len;
            carry += total;
            if (j < tf.ne) {
                m.sadj[j] = base + sh - (uint32_t)r0c;
                tma_load_1d(stage_ptr(st) + base, reinterpret_cast<const void *>(src_lo), len, &s_bar[st]);
            }
        }
        if (tid == 0) {
            m.ne = tf.ne;
            m.tile_len = tile_len;
            m.T0 = T0;
            mbar_expect_tx(&s_bar[st], carry); // one arrival: the phase completes when all `carry` bytes have landed
        }
    };

    uint4 recA[kGtPer], recB[kGtPer];
    unsigned long long srcA[kGtPer], srcB[kGtPer];
    uint32_t tile = blockIdx.x;
    TF tf_cur = load_tf(tile), tf_nxt = load_tf(tile + G);
    load_recs(tf_cur, recA, srcA);
    publish(0, tile, tf_cur, recA, srcA);
    load_recs(tf_nxt, recA, srcA);        // metadata of the NEXT tile rides in registers
    TF tf_nn = load_tf(tile + 2 * G);

    for (uint32_t q = 0;; q++) {
        const uint32_t st = q & 1;
        const bool has_next = tile + G < n_tiles;
        if (has_next) publish(st ^ 1, tile + G, tf_nxt, recA, srcA);
        load_recs(tf_nn, recB, srcB);                 // tile q + 2
        const TF tf_n3 = load_tf(tile + 3 * G);       // tile q + 3
        __syncthreads();                              // meta[st] was written one iteration ago by other threads
        while (!mbar_try_wait(&s_bar[st], (q >> 1) & 1)) {}

        const GtMeta &m = *meta_ptr(st);
        const uint8_t *sd = stage_ptr(st);
        const uint32_t ne = m.ne, tile_len = m.tile_len;
        uint8_t *dst_tile = p.out_data + m.T0;

        // ---- copy: warp w owns bytes [w * 2 KB, (w + 1) * 2 KB) of the tile, 1 KB (32 lanes x 32 bytes) at a time
        const int sub0 = (int)(warp * (uint32_t)(kG32Vpt * 1024));
        if ((uint32_t)sub0 < tile_len) {
            uint32_t j = 0;
            for (uint32_t base = 0; base + 1 < ne; base += 32) {
                const uint32_t i = base + lane;
                j += __popc(__ballot_sync(0xFFFFFFFFu, i + 1 < ne && m.r1[i] <= sub0));
            }
            const uint32_t lanes_le = 0xFFFFFFFFu >> (31 - lane);
#pragma unroll
            for (int k = 0; k < kG32Vpt; k++) {
                const int cb = sub0 + k * 1024;
                const int b0 = cb + (int)lane * 32;
                const uint32_t i = j + lane;
                const int r1 = i + 1 < ne ? m.r1[i] : 0x7FFFFFFF;
                const bool ends_here = r1 <= cb + 1024;
                const uint32_t t = (uint32_t)((ends_here ? r1 : cb + 32) - cb + 31) >> 5;
                const uint32_t ends = __reduce_or_sync(0xFFFFFFFFu, (ends_here && t < 32) ? (1u << t) : 0u);
                const uint32_t cnt = __popc(ends & lanes_le);
                const uint32_t adv = __popc(__ballot_sync(0xFFFFFFFFu, ends_here));
                const uint32_t e = j + cnt;
                j += adv;
                const int r1e = m.r1[e];
                const bool pure = (uint32_t)b0 + 32 <= tile_len && b0 + 32 <= r1e;
                if (pure) { // divergence is cheap here: nothing is in flight, the operands are in shared memory
                    const uint32_t sa = m.sadj[e] + (uint32_t)b0;
                    const uint32_t sh = sa & 15u;
                    const uint4 *sv = reinterpret_cast<const uint4 *>(sd + (sa - sh));
                    const uint4 A = sv[0], B = sv[1], C = sv[sh ? 2 : 1];
                    uint32_t o[8];
                    realign32(A, B, C, sh, o);
                    stg256(dst_tile + b0, o);
                }
            }
        }

        // ---- the 32-byte block that holds the last byte of entry j (unless j ends on a block boundary): its two halves
        for (uint32_t j = tid; j < ne; j += NT) {
            const int r1 = m.r1[j];
            if (r1 <= 0 || (r1 & 31) == 0 || r1 > (int)tile_len) continue;
            const bool has_nx = j + 1 < ne;
#pragma unroll
            for (int half = 0; half < 2; half++) {
                const uint32_t b0 = ((uint32_t)r1 & ~31u) + 16u * half;
                if (b0 >= tile_len) continue;
                const int t = r1 - (int)b0;
                uint4 o;
                if (t >= 16) {
                    o = lds16_any(sd, m.sadj[j] + b0, 16);
                } else if (t <= 0) {
                    if (!has_nx) continue;
                    o = lds16_any(sd, m.sadj[j + 1] + b0, 16);
                } else {
                    o = lds16_any(sd, m.sadj[j] + b0, (uint32_t)t);
                    if (b0 + 16 <= tile_len) {
                        const uint4 H = lds16_any(sd, m.sadj[j + 1] + (uint32_t)r1, 16);
                        const uint4 HU = realign16_sel(make_uint4(0, 0, 0, 0), H, 16 - (uint32_t)t);
                        const uint32_t wfull = (uint32_t)t >> 2, bits = ((uint32_t)t & 3) * 8;
                        const uint32_t mmix = bits ? (0xFFFFFFFFu >> (32 - bits)) : 0u;
                        uint32_t ow[4] = {o.x, o.y, o.z, o.w}, hw[4] = {HU.x, HU.y, HU.z, HU.w};
#pragma unroll
                        for (uint32_t qq = 0; qq < 4; qq++) {
                            const uint32_t mk = qq < wfull ? 0xFFFFFFFFu : (qq == wfull ? mmix : 0u);
                            ow[qq] = (ow[qq] & mk) | (hw[qq] & ~mk);
                        }
                        o = make_uint4(ow[0], ow[1], ow[2], ow[3]);
                    } else { // ragged end of the whole stream
                        const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
                        for (int b = 0; b < t; b++) dst_tile[b0 + b] = (uint8_t)(ow[b >> 2] >> ((b & 3) * 8));
                        continue;
                    }
                }
                reinterpret_cast<uint4 *>(dst_tile)[b0 >> 4] = o;
            }
        }

        // ---- bloom (fused epilogue): entries whose first byte lies in this tile; keys from shared memory when they are
        // wholly staged (an entry that runs into the next tile may have its key cut off: global loads then)
        if (p.bloom.words != nullptr && p.hash_rec == nullptr && !p.bloom_elsewhere) {
            for (uint32_t j = tid; j < ne; j += NT) {
                const int r0 = m.r0[j];
                if (r0 < 0 || r0 >= (int)kGatherTileBytes) continue;
                const uint64_t klen = m.ks[j] - 8;
                uint64_t h0, h1;
                if ((uint64_t)r0 + 16 + klen <= (uint64_t)tile_len) {
                    const uint8_t *key = sd + (m.sadj[j] + (uint32_t)r0 + 8u);
                    sip13_pair_vec_u8(p.bloom.sip, klen, [key](uint64_t qq) {
                        const uintptr_t a = reinterpret_cast<uintptr_t>(key + 8 * qq);
                        const uint64_t *w = reinterpret_cast<const uint64_t *>(a & ~uintptr_t(7));
                        const uint32_t shb = (uint32_t)(a & 7) * 8;
                        const uint64_t lo = w[0];
                        return shb ? (lo >> shb) | (w[1] << (64 - shb)) : lo;
                    }, &h0, &h1);
                } else {
                    const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)(m.adj[j] + (unsigned long long)r0)) + 8;
                    sip13_pair_vec_u8(p.bloom.sip, klen, [key](uint64_t qq) { return ld_u64_unaligned(key + 8 * qq); }, &h0, &h1);
                }
                uint32_t *words = p.bloom.words;
                bloom_probe_all(h0, h1, p.bloom.k_num, p.bloom.bits, p.bloom.bits_magic,
                                [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
            }
        }

        if (!has_next) break;
        __syncthreads(); // everyone is done with stage st and meta[st]: the next iteration's publish overwrites st ^ 1's peer
        tile += G;
        tf_nxt = tf_nn;
        tf_nn = tf_n3;
#pragma unroll
        for (int k = 0; k < kGtPer; k++) { recA[k] = recB[k]; srcA[k] = srcB[k]; }
    }
}

// ------------------------------------------------------------------------------------
// K5, persistent with prefetched metadata (k_gather32's copy, different skeleton).  In k_gather32 a CTA's life is a chain
// of memory round trips -- tile_first -> out_index / src_ptr -> payload -> boundary / key bytes -- and only the other
// resident CTAs cover them.  Here a CTA keeps going tile after tile, and the first two links of the NEXT tile's chain run
// while the current tile is copied: the tile_first pair two tiles ahead travels in registers, the out_index / src_ptr
// records of the next tile arrive in shared memory through cp.async (LDGSTS: no registers held).  What is left on a
// tile's critical path is one payload round trip.

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async8(void *smem_dst, const void *gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}

#ifndef DBEEL_GP_CTAS
#define DBEEL_GP_CTAS 10
#endif
__global__ void __launch_bounds__(kGatherThreads, DBEEL_GP_CTAS) k_gather_p(Params p) {
    pdl_trigger();
    pdl_wait();
    constexpr int NT = kGatherThreads;
    __shared__ __align__(16) uint4 s_rawi[2][kGatherMaxEntries];
    __shared__ __align__(8) unsigned long long s_raws[2][kGatherMaxEntries];
    __shared__ unsigned long long s_adj[kGatherMaxEntries];
    __shared__ int s_r0[kGatherMaxEntries], s_r1[kGatherMaxEntries];
    __shared__ uint32_t s_ks[kGatherMaxEntries];
    const Ctl *c = p.ctl;
    const unsigned long long out_len = c->out_data_len;
    const uint32_t out_items = c->out_items;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t n_tiles = (uint32_t)((out_len + kGatherTileBytes - 1) / kGatherTileBytes);
    const uint32_t G = gridDim.x;
    uint32_t tile = blockIdx.x;
    if (tile >= n_tiles) return;
    const bool hash_here = p.bloom.words != nullptr && p.hash_rec == nullptr && !p.bloom_elsewhere;

    auto tf_lo = [&](uint32_t t) -> uint32_t { return t < n_tiles ? __ldg(&p.tile_first[t]) : 0u; };
    auto tf_ne = [&](uint32_t t, uint32_t lo) -> uint32_t {
        if (t >= n_tiles) return 0u;
        const uint32_t hi = t + 1 < n_tiles ? __ldg(&p.tile_first[t + 1]) : out_items - 1;
        return hi - lo + 1;
    };
    auto prefetch = [&](uint32_t buf, uint32_t lo, uint32_t ne) {
        for (uint32_t j = tid; j < ne; j += NT) {
            cp_async16(&s_rawi[buf][j], &p.out_index[lo + j]);
            cp_async8(&s_raws[buf][j], &p.src_ptr[lo + j]);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    uint32_t lo0 = tf_lo(tile), ne0 = tf_ne(tile, lo0);
    prefetch(0, lo0, ne0);
    uint32_t lo1 = tf_lo(tile + G), ne1 = tf_ne(tile + G, lo1);

    for (uint32_t q = 0;; q++) {
        const uint32_t buf = q & 1;
        const bool has_next = tile + G < n_tiles;
        prefetch(buf ^ 1, lo1, ne1); // an empty group when there is no next tile
        const uint32_t lo2 = tf_lo(tile + 2 * G), ne2 = tf_ne(tile + 2 * G, lo2); // consumed one iteration from now
        asm volatile("cp.async.wait_group 1;" ::: "memory"); // everything but the group just committed has landed
        __syncthreads();

        const unsigned long long T0 = (unsigned long long)tile * kGatherTileBytes;
        const uint32_t tile_len = out_len - T0 < kGatherTileBytes ? (uint32_t)(out_len - T0) : (uint32_t)kGatherTileBytes;
        const uint32_t ne = ne0;
        for (uint32_t j = tid; j < ne; j += NT) {
            const uint4 rec = s_rawi[buf][j];
            const unsigned long long d0 = ((unsigned long long)rec.x | ((unsigned long long)rec.y << 32)) - p.out_offset_base;
            const long long r0 = (long long)d0 - (long long)T0;
            const long long r1 = r0 + (long long)rec.w;
            s_adj[j] = s_raws[buf][j] - (unsigned long long)r0;
            s_r0[j] = r0 < -0x7FFFFFFFll ? -0x7FFFFFFF : (int)r0;
            s_r1[j] = r1 > 0x7FFFFFFFll ? 0x7FFFFFFF : (int)r1;
            if (hash_here) s_ks[j] = rec.z;
        }
        __syncthreads();

        // ---- copy (k_gather32's): warp w owns bytes [w * 2 KB, (w + 1) * 2 KB) of the tile, 1 KB at a time
        uint8_t *dst_tile = p.out_data + T0;
        const int sub0 = (int)(warp * (uint32_t)(kG32Vpt * 1024));
        if ((uint32_t)sub0 < tile_len) {
            uint32_t j = 0;
            for (uint32_t base = 0; base + 1 < ne; base += 32) {
                const uint32_t i = base + lane;
                j += __popc(__ballot_sync(0xFFFFFFFFu, i + 1 < ne && s_r1[i] <= sub0));
            }
            uint4 A[kG32Vpt], B[kG32Vpt], C[kG32Vpt];
            uint32_t sh[kG32Vpt];
            bool pure[kG32Vpt];
            const uint32_t lanes_le = 0xFFFFFFFFu >> (31 - lane);
#pragma unroll
            for (int k = 0; k < kG32Vpt; k++) {
                const int cb = sub0 + k * 1024;
                const int b0 = cb + (int)lane * 32;
                const uint32_t i = j + lane;
                const int r1 = i + 1 < ne ? s_r1[i] : 0x7FFFFFFF;
                const bool ends_here = r1 <= cb + 1024;
                const uint32_t t = (uint32_t)((ends_here ? r1 : cb + 32) - cb + 31) >> 5;
                const uint32_t ends = __reduce_or_sync(0xFFFFFFFFu, (ends_here && t < 32) ? (1u << t) : 0u);
                const uint32_t cnt = __popc(ends & lanes_le);
                const uint32_t adv = __popc(__ballot_sync(0xFFFFFFFFu, ends_here));
                const uint32_t e = j + cnt;
                j += adv;
                const int r1e = s_r1[e];
                pure[k] = (uint32_t)b0 + 32 <= tile_len && b0 + 32 <= r1e;
                const int bl = b0 + 32 <= r1e ? b0 : r1e - 32;
                const uintptr_t sa = (uintptr_t)(s_adj[e] + (unsigned long long)(long long)bl);
                sh[k] = (uint32_t)(sa & 15);
                const uint4 *sv = reinterpret_cast<const uint4 *>(sa - sh[k]);
                A[k] = __ldg(sv);
                B[k] = __ldg(sv + 1);
                C[k] = __ldg(sh[k] ? sv + 2 : sv + 1);
            }
#pragma unroll
            for (int k = 0; k < kG32Vpt; k++) {
                if (pure[k]) {
                    uint32_t o[8];
                    realign32(A[k], B[k], C[k], sh[k], o);
                    stg256(dst_tile + sub0 + k * 1024 + (int)lane * 32, o);
                }
            }
        }

        // ---- the 32-byte block that holds the last byte of entry j: its two halves
        for (uint32_t j = tid; j < ne; j += NT) {
            const int r1 = s_r1[j];
            if (r1 <= 0 || (r1 & 31) == 0 || r1 > (int)tile_len) continue;
            const bool has_nx = j + 1 < ne;
#pragma unroll
            for (int half = 0; half < 2; half++) {
                const uint32_t b0 = ((uint32_t)r1 & ~31u) + 16u * half;
                if (b0 >= tile_len) continue;
                const int t = r1 - (int)b0;
                uint4 o;
                if (t >= 16) {
                    o = ld16_any((uintptr_t)(s_adj[j] + b0), 16);
                } else if (t <= 0) {
                    if (!has_nx) continue;
                    o = ld16_any((uintptr_t)(s_adj[j + 1] + b0), 16);
                } else {
                    o = ld16_any((uintptr_t)(s_adj[j] + b0), (uint32_t)t);
                    if (b0 + 16 <= tile_len) {
                        const uint4 H = ld16_any((uintptr_t)(s_adj[j + 1] + (unsigned long long)(long long)r1), 16);
                        const uint4 HU = realign16_sel(make_uint4(0, 0, 0, 0), H, 16 - (uint32_t)t);
                        const uint32_t wfull = (uint32_t)t >> 2, bits = ((uint32_t)t & 3) * 8;
                        const uint32_t mmix = bits ? (0xFFFFFFFFu >> (32 - bits)) : 0u;
                        uint32_t ow[4] = {o.x, o.y, o.z, o.w}, hw[4] = {HU.x, HU.y, HU.z, HU.w};
#pragma unroll
                        for (uint32_t qq = 0; qq < 4; qq++) {
                            const uint32_t mk = qq < wfull ? 0xFFFFFFFFu : (qq == wfull ? mmix : 0u);
                            ow[qq] = (ow[qq] & mk) | (hw[qq] & ~mk);
                        }
                        o = make_uint4(ow[0], ow[1], ow[2], ow[3]);
                    } else {
                        const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
                        for (int b = 0; b < t; b++) dst_tile[b0 + b] = (uint8_t)(ow[b >> 2] >> ((b & 3) * 8));
                        continue;
                    }
                }
                reinterpret_cast<uint4 *>(dst_tile)[b0 >> 4] = o;
            }
        }

        // ---- bloom (fused epilogue) unless it runs elsewhere
        if (hash_here) {
            for (uint32_t j = tid; j < ne; j += NT) {
                const int r0 = s_r0[j];
                if (r0 < 0 || r0 >= (int)kGatherTileBytes) continue;
                const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)(s_adj[j] + (unsigned long long)r0)) + 8;
                const uint64_t klen = s_ks[j] - 8;
                uint64_t h0, h1;
                sip13_pair_vec_u8(p.bloom.sip, klen, [key](uint64_t qq) { return ld_u64_unaligned(key + 8 * qq); }, &h0, &h1);
                uint32_t *words = p.bloom.words;
                bloom_probe_all(h0, h1, p.bloom.k_num, p.bloom.bits, p.bloom.bits_magic,
                                [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
            }
        }

        if (!has_next) break;
        __syncthreads(); // s_adj / s_r0 / s_r1 and raw buffer `buf` are free again
        tile += G;
        lo0 = lo1; ne0 = ne1;
        lo1 = lo2; ne1 = ne2;
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Job header down / control block up without a copy engine: the pinned block is mapped into the GPU's address space.
__global__ void __launch_bounds__(256) k_copy_words(uint32_t *dst, const uint32_t *src_host, uint32_t n) {
    pdl_trigger();
    pdl_wait();
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    if (i < n) dst[i] = src_host[i];
}

__global__ void __launch_bounds__(256) k_publish(uint32_t *dst_host, const uint32_t *ctl, uint32_t n_ctl, uint32_t *dst2_host,
                                                 const uint32_t *table, uint32_t n_table) {
    pdl_trigger();
    pdl_wait();
    for (uint32_t i = threadIdx.x; i < n_ctl; i += 256) dst_host[i] = ctl[i];
    for (uint32_t i = threadIdx.x; i < n_table; i += 256) dst2_host[i] = table[i];
    __threadfence_system(); // visible to the host before the stream reports completion
}

// .bloom framing around the bit vector (bincode of bloomfilter::Bloom, DESIGN.md):
//   u64 n_words | u32 words[n_words] | u64 nbits | u64 bitmap_bits | u32 k_num | 2 x SipHasher13
__global__ void k_bloom_frame(uint8_t *file, uint64_t n_words, BloomParams b) {
    pdl_trigger();
    pdl_wait();
    if (threadIdx.x || blockIdx.x) return;
    uint32_t *w = reinterpret_cast<uint32_t *>(file);
    auto put64 = [&](uint64_t word_idx, uint64_t v) {
        w[word_idx] = (uint32_t)v;
        w[word_idx + 1] = (uint32_t)(v >> 32);
    };
    put64(0, n_words);
    uint64_t t = 2 + n_words; // u32 index of the trailer
    put64(t, b.bits);
    put64(t + 2, b.bits);
    w[t + 4] = b.k_num;
    t += 5;
    for (int h = 0; h < 2; h++) {
        uint64_t k0 = b.sip[2 * h], k1 = b.sip[2 * h + 1];
        put64(t, k0);
        put64(t + 2, k1);
        put64(t + 4, 0);                          // length
        put64(t + 6, k0 ^ 0x736f6d6570736575ULL); // v0
        put64(t + 8, k0 ^ 0x6c7967656e657261ULL); // v2
        put64(t + 10, k1 ^ 0x646f72616e646f6dULL); // v1
        put64(t + 12, k1 ^ 0x7465646279746573ULL); // v3
        put64(t + 14, 0);                         // tail
        put64(t + 16, 0);                         // ntail
        t += 18;
    }
}

// Single job, filter filled NEXT TO the gather instead of inside it: one thread per merged position, survivors only
// (res[i].w != 0), key bytes from the entry's source (one 64-byte granule for ordinary keys).  Launched on the engine's
// second stream right after k_resolve, so its random reads and SipHash rounds overlap k_emit and the payload copy -- the
// gather is the kernel with no issue slot and no latency slack to spare, this one is all latency.
__global__ void __launch_bounds__(256) k_bloom_res(Params p, const uint4 *res) {
    pdl_trigger();
    pdl_wait();
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    if (i >= p.ctl->span) return;
    const uint4 it = __ldg(&res[i]);
    if (it.w == 0) return;
    const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)((unsigned long long)it.x | ((unsigned long long)it.y << 32))) + 8;
    uint64_t h0, h1;
    sip13_pair_vec_u8(p.bloom.sip, (uint64_t)(it.z - 8), [key](uint64_t q) { return ld_u64_unaligned_narrow(key + 8 * q); }, &h0, &h1);
    uint32_t *words = p.bloom.words;
    bloom_probe_all(h0, h1, p.bloom.k_num, p.bloom.bits, p.bloom.bits_magic,
                    [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
}

// compact-many: the filters are per job (own size, own seed), so they are filled by a pass of their own over the output
// entries instead of the gather's fused epilogue (which stays untouched for the single-job path): one thread per entry,
// job = last one whose first output entry is <= e (k_flush_table's rows), key bytes from the entry's source.
__global__ void __launch_bounds__(256) k_bloom_many(Params p) {
    pdl_trigger();
    pdl_wait();
    const uint32_t e = blockIdx.x * 256u + threadIdx.x;
    if (e >= p.ctl->out_items) return;
    uint32_t lo = 0, hi = p.n_groups;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (p.mem_table[2 * mid + 1] <= e) lo = mid; else hi = mid;
    }
    const BloomParams bp = p.groups[lo].bloom;
    uint32_t *words = bp.words;
    if (words == nullptr) return;
    const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)p.src_ptr[e]) + 8;
    const uint64_t klen = p.out_index[e].z - 8;
    uint64_t h0, h1;
    sip13_pair_vec_u8(bp.sip, klen, [key](uint64_t q) { return ld_u64_unaligned(key + 8 * q); }, &h0, &h1);
    bloom_probe_all(h0, h1, bp.k_num, bp.bits, bp.bits_magic,
                    [words](uint64_t bit) { atomicOr(&words[bit >> 5], 1u << (bit & 31)); });
}

// compact-many: one frame per job that has a filter
__global__ void __launch_bounds__(128) k_bloom_frames(const GroupDesc *groups, uint32_t n_groups) {
    pdl_trigger();
    pdl_wait();
    const uint32_t g = blockIdx.x * 128u + threadIdx.x;
    if (g >= n_groups) return;
    const BloomParams b = groups[g].bloom;
    if (b.words == nullptr) return;
    uint32_t *w = b.words - 2; // the file starts 8 bytes before the bit vector
    const uint64_t n_words = (b.bits + 31) / 32;
    auto put64 = [&](uint64_t word_idx, uint64_t v) {
        w[word_idx] = (uint32_t)v;
        w[word_idx + 1] = (uint32_t)(v >> 32);
    };
    put64(0, n_words);
    uint64_t t = 2 + n_words;
    put64(t, b.bits);
    put64(t + 2, b.bits);
    w[t + 4] = b.k_num;
    t += 5;
    for (int h = 0; h < 2; h++) {
        const uint64_t k0 = b.sip[2 * h], k1 = b.sip[2 * h + 1];
        put64(t, k0);
        put64(t + 2, k1);
        put64(t + 4, 0);
        put64(t + 6, k0 ^ 0x736f6d6570736575ULL);
        put64(t + 8, k0 ^ 0x6c7967656e657261ULL);
        put64(t + 10, k1 ^ 0x646f72616e646f6dULL);
        put64(t + 12, k1 ^ 0x7465646279746573ULL);
        put64(t + 14, 0);
        put64(t + 16, 0);
        t += 18;
    }
}

// DBEEL_FLAG_VERIFY_SORTED: every valid entry i > 0 of a run must have key[i-1] < key[i].
__global__ void __launch_bounds__(256) k_verify_sorted(Params p) {
    pdl_trigger();
    pdl_wait();
    uint32_t g = blockIdx.x * 256u + threadIdx.x;
    if (g >= p.n_total) return;
    uint32_t r = find_run(p, g);
    uint32_t i = g - p.runs[r].base;
    if (i == 0 || i >= p.first_bad[r]) return;
    if (full_key_cmp(p, g - 1, g, 0) >= 0) atomicOr(&p.ctl->flags, kFlagVerifyFailed);
}

// ------------------------------------------------------------------------------------
// DBEEL_FLAG_REFERENCE_READER, slow path: some index record disagreed with the data (k_extract<.., true> pass 0).  The
// reference's reader never notices -- it takes full_size from the index and everything else from the next full_size
// bytes of .data -- so the job continues on a canonical copy of the index that says what that reader sees:
//   offset = running sum of full_size (the stream cursor), key_size = 8 + the length prefix found at the cursor.
// One CTA per run walks it in 1024-record chunks with a carried cursor (a rare path: corrupt or foreign index files).
__global__ void __launch_bounds__(1024) k_ref_repair(Params p) {
    pdl_trigger();
    pdl_wait();
    __shared__ unsigned long long s_b[32];
    __shared__ uint32_t s_c[32];
    if (!(p.ctl->flags & kFlagIndexDiffers)) return;
    const RunDesc rd = p.runs[blockIdx.x];
    unsigned long long carry = rd.off_base;
    for (uint32_t base = 0; base < rd.n_in; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        uint4 rec = make_uint4(0, 0, 0, 0);
        if (i < rd.n_in) rec = __ldg(&rd.index[i]);
        unsigned long long vb = rec.w, tb;
        uint32_t vc = 0, tc;
        __syncthreads(); // s_b / s_c of the previous chunk are still being read
        block_excl_scan_1024(vb, vc, s_b, s_c, &tb, &tc);
        const unsigned long long cur = carry + vb;
        if (i < rd.n_in) {
            uint32_t ks = rec.z;
            if (cur >= rd.off_base && cur <= rd.data_len && rd.data_len - cur >= 8) {
                const uint64_t klen = ld_u64_unaligned(rd.data + cur);
                ks = klen > 0xFFFFFFF0ull ? 0xFFFFFFFFu : (uint32_t)klen + 8u;
            }
            p.fix_index[rd.base + i] = make_uint4((uint32_t)cur, (uint32_t)(cur >> 32), ks, rec.w);
        }
        carry += tb;
    }
}

// ... then the job state goes back to "nothing validated yet", now reading the canonical index
__global__ void k_ref_reset(Params p) {
    pdl_trigger();
    pdl_wait();
    Ctl *c = p.ctl;
    if (!(c->flags & kFlagIndexDiffers)) return;
    RunDesc *runs = const_cast<RunDesc *>(p.runs);
    for (uint32_t r = threadIdx.x; r < p.n_runs; r += blockDim.x) {
        runs[r].index = p.fix_index + runs[r].base;
        p.first_bad[r] = runs[r].n_in;
        p.first_mismatch[r] = 0xFFFFFFFFu;
    }
    __syncthreads();
    if (threadIdx.x == 0) c->flags = (c->flags & ~(kFlagIndexDiffers | kFlagTruncated)) | kFlagRepaired;
}

} // namespace dbeel
