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

constexpr unsigned long long kGatherTileBytes = 16ull * kGatherThreads * kGatherVecsPerThread; // 8 KB of output per CTA
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
    uint32_t *tile_first;        // [ceil(data bytes / kGatherTileBytes) + 2] entry holding each gather tile's first byte
    uint32_t tile_first_n;       // gather tiles the buffers were sized for (sparse batches: the caller's bound may be too low)
    unsigned long long data_bound; // .data bytes the job checked against out->data_cap: k_gather_h writes nothing at or past it
    unsigned long long out_offset_base; // .data bytes written by earlier key-range partitions of the same output file
    BloomParams bloom;
    // fused last merge level + resolve + emit (k_merge_final, single jobs): chained scan of the tiles' (bytes, entries), decoupled look-back
    uint32_t fin_tile;   // k_merge_final: nominal records per tile of the LAST level (< kMergeTile: room for the extensions), 0 = off
    uint32_t *part_ext;  // [boundaries of the last level] records with the boundary's key that follow it in A (bits 0-7) and B (8-15)
    unsigned long long *scan_state; // [k_merge_final tiles][2]: {status << 62 | bytes, status << 32 | entries}, zeroed per job
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
template <bool kNarrow, bool kRef, bool kPersist = false>
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

template <bool kNarrow>
__global__ void __launch_bounds__(kResolveThreads, DBEEL_RESOLVE_MINB) k_resolve(Params p, const Rec *m, uint4 *res) {
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
    const uint32_t i0 = blockIdx.x * NT;
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

    uint32_t keep = 0, ks = 0, fs = 0;
    unsigned long long src = 0;
    if (p.mode_flush) {
        // Arrival batches: the winner of a group of equal keys is simply its LAST member (RedBlackTree::set replaces in place,
        // lib.rs:509-511), and every member knows locally whether it is the last one.  No walk over the group: a hot key of a
        // Zipf stream fills hundreds of consecutive positions of a memtable, and a head thread stepping through them one
        // dependent load at a time dominated the whole flush of a Zipf stream.
        if (active && !eq_next) {
            keep = 1; // tombstones are ordinary entries of a flush (lsm_tree.rs:790-795)
            ks = s_ks[tid]; fs = s_fs[tid]; src = s_entry[tid];
        }
    } else if (active && !eq_prev) { // head of its group
        uint32_t w = tid; // winner so far, as an index into this tile's shared arrays
        ks = s_ks[tid]; fs = s_fs[tid]; src = s_entry[tid];
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
                    if (better) { ks = ck.klen + 8; fs = ck.full_size; src = (unsigned long long)(uintptr_t)ck.entry; }
                    gj++;
                    if (gj >= lim_hi) break;
                    if (!key_equal(p, skip, nx, ld_rec(&m[gj]))) break;
                }
            }
        }
        bool tomb = fs == ks + 24;
        keep = (keep_tombstones || p.mode_flush || !tomb) ? 1u : 0u;
    }
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
}


// ------------------------------------------------------------------------------------
// K4b: offsets.  The survivor at merged position i becomes output entry `count before i`, at
// .data offset `bytes before i` (entry_writer.rs:81-86: offset = running sum of full_size).
// No inter-CTA waiting: (1) the per-tile aggregates are scanned in chunks of 1024 tiles, (2) one
// CTA scans the chunk totals, (3) every tile rescans its 256 records locally and emits
// out_index (the output .index file itself), src_ptr, and -- for every gather tile (kGatherTileBytes)
// of the output .data stream -- the entry that holds the tile's first byte (tile_first).

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
