// merge_final.cuh -- the LAST merge level, resolve, the offsets scan and the .index writes of a single compaction in ONE
// persistent kernel (round 2).
//
// Round 1 ran them as five kernels: k_merge_tma (last level) -> k_resolve -> k_scan_tiles -> k_scan_chunks -> k_emit, with the
// merged records and the per-position results (`res`) making a round trip through HBM between them (4 x 16 bytes per input
// entry) and two latency-bound launches of one thread per record.  Here a tile of the last level stays in shared memory
// after it has been merged:
//
//   TMA (2 bulk copies, mbarrier)   A / B ranges of the tile, plus the record on either side of each range (the neighbours
//                                   that decide whether a group of equal keys crosses the tile's edges)
//   merge-path, 7 records / thread  sorted tile in shared memory (as k_merge_tma)
//   resolve                         7 independent chains per thread: index record by gid (64-byte granule), timestamp only
//                                   for members of a group; the head of a group picks max (timestamp, run position) over
//                                   shared memory (lsm_tree.rs:1036-1066, mod.rs:75-81) and applies the tombstone rule
//   scan                            (bytes, entries) of the tile's survivors; chained scan over the tiles, the aggregate
//                                   published at once, the one-warp look-back deferred by one tile (see the tile loop)
//   emit                            output .index records, src_ptr, tile_first (entry_writer.rs:76-86) from the survivors
//                                   kept in shared memory, one tile later
//
// What no longer exists: the last level's 16 B/entry write, k_resolve's 16 B read + 16 B `res` write, k_emit's 16 B read,
// three kernel boundaries and the two scan kernels.
#pragma once
#include "kernels.cuh"

namespace dbeel {

constexpr int kFinThreads = kMergeThreads;
constexpr int kFinVT = kMergeVT;
constexpr int kFinTile = kMergeTile;           // capacity of a tile: 7 records per thread
constexpr int kFinNominal = kFinTile - 64;     // nominal tile (k_merge_partition's split points); + up to 31 + 31 records of a straddling group
constexpr int kFinBufRecs = kFinTile + 8;      // A_prev | A | A_next | B_prev | B | B_next, + slack
constexpr int kFinMaxRunsSmem = 64;            // run tables (base / index / data) cached in shared memory up to this many runs
#ifndef DBEEL_FIN_CTAS
#define DBEEL_FIN_CTAS 2
#endif
constexpr uint32_t kFinSmem = 2u * kFinBufRecs * 16u + 2u * kFinTile * 8u + (uint32_t)kFinTile + 16u;

// Measurement builds only (`python -m dbeel_b200._build --variant phases DBEEL_FIN_PHASES`): thread 0 of every CTA books the
// clock64() time between consecutive marks -- most taken right after a CTA-wide wait, so such a phase is its slowest
// thread's -- and the last CTA of a launch prints the sums over all CTAs, then clears them.  Outputs are those of the
// normal build.
#ifdef DBEEL_FIN_PHASES
constexpr int kFinPhases = 8;
__device__ unsigned long long g_fin_phase[kFinPhases];
__device__ unsigned int g_fin_done;
#define FIN_PH_DECL unsigned long long ph_acc[kFinPhases] = {}; long long ph_t = clock64();
#define FIN_PH(k) do { if (tid == 0) { const long long ph_n = clock64(); ph_acc[k] += (unsigned long long)(ph_n - ph_t); ph_t = ph_n; } } while (0)
__device__ __forceinline__ void fin_phase_flush(const unsigned long long *acc, uint32_t n_tiles) { // thread 0
    for (int k = 0; k < kFinPhases; k++) atomicAdd(&g_fin_phase[k], acc[k]);
    __threadfence();
    if (atomicAdd(&g_fin_done, 1u) + 1 == (gridDim.x < n_tiles ? gridDim.x : n_tiles)) { // CTAs without a tile return early
        __threadfence();
        unsigned long long v[kFinPhases], tot = 0;
        for (int k = 0; k < kFinPhases; k++) { v[k] = atomicExch(&g_fin_phase[k], 0ull); tot += v[k]; }
        g_fin_done = 0;
        printf("fin_phases ctas=%u cycles=%llu tma=%llu merge=%llu index_issue=%llu index_wait=%llu lookback=%llu emit=%llu "
               "ts_wait=%llu heads_scan=%llu\n", gridDim.x, tot, v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
    }
}
#else
#define FIN_PH_DECL
#define FIN_PH(k) do {} while (0)
#endif

struct FinDesc {
    uint32_t a_src, n_a, b_src, n_b; // record offsets into src, counts
    uint32_t a_end, b_end;           // one past the last record of segment A / B (absolute)
    uint32_t diag0;                  // merged position of the tile's first record, relative to the pair's output
    uint32_t nb;                     // bit 0: A[a0-1] exists, 1: A[a1] exists, 2: B[b0-1] exists, 3: B[b1] exists
};

// Decoupled look-back of tile t > 0 by one warp: lane l reads the state of predecessors t-1-4l ... t-4-4l (all four loads in
// flight together), waits only for a predecessor that has published nothing yet, and the walk stops at the nearest one that
// holds an inclusive prefix.  (eb, ec) = bytes and entries of every tile before t, in every lane.
__device__ __forceinline__ void fin_lookback(const unsigned long long *scan_state, uint32_t t, uint32_t lane, unsigned long long &eb,
                                             uint32_t &ec) {
    constexpr int kPer = 4;
    eb = 0;
    ec = 0;
    for (int base = (int)t - 1;; base -= 32 * kPer) {
        unsigned long long vb[kPer], vc[kPer];
#pragma unroll
        for (int k = 0; k < kPer; k++) {
            const int idx = base - (int)lane * kPer - k;
            vb[k] = kScanPrefix << 62; // tiles before the first one: a prefix of nothing
            vc[k] = kScanPrefix << 32;
            if (idx >= 0) {
                vc[k] = ld_volatile_u64(scan_state + 2ull * (uint32_t)idx + 1);
                vb[k] = ld_volatile_u64(scan_state + 2ull * (uint32_t)idx);
            }
        }
        bool found = false;
        unsigned long long sb = 0;
        uint32_t sc = 0;
#pragma unroll
        for (int k = 0; k < kPer; k++) {
            const int idx = base - (int)lane * kPer - k;
            // each word says what it holds: both at the same stage, or read the pair again
            while ((vc[k] >> 32) == 0 || (vc[k] >> 32) != (vb[k] >> 62)) {
                vc[k] = ld_volatile_u64(scan_state + 2ull * (uint32_t)idx + 1);
                vb[k] = ld_volatile_u64(scan_state + 2ull * (uint32_t)idx);
            }
            if (!found) {
                sb += vb[k] & ((1ull << 62) - 1);
                sc += (uint32_t)vc[k];
                found = (vc[k] >> 32) == kScanPrefix;
            }
        }
        const uint32_t fm = __ballot_sync(0xFFFFFFFFu, found);
        const uint32_t first = fm ? (uint32_t)__ffs((int)fm) - 1u : 32u; // the lane holding the nearest prefix
        if (lane > first) { sb = 0; sc = 0; }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            sb += __shfl_xor_sync(0xFFFFFFFFu, sb, o);
            sc += __shfl_xor_sync(0xFFFFFFFFu, sc, o);
        }
        eb += sb;
        ec += sc;
        if (fm) return;
    }
}

template <bool kNarrow>
__global__ void __launch_bounds__(kFinThreads, DBEEL_FIN_CTAS) k_merge_final(const __grid_constant__ Params p, uint32_t level, const Rec *src) {
    constexpr int NT = kFinThreads, VT = kFinVT;
    extern __shared__ __align__(128) uint8_t f_raw[];
    Rec *bufs[2] = {reinterpret_cast<Rec *>(f_raw), reinterpret_cast<Rec *>(f_raw) + kFinBufRecs};
    unsigned long long *s_tlo = reinterpret_cast<unsigned long long *>(f_raw + 2u * kFinBufRecs * 16u);
    unsigned long long *s_thi = s_tlo + kFinTile;
    uint8_t *s_flag = reinterpret_cast<uint8_t *>(s_thi + kFinTile); // bit 0: same key as the next merged record
    __shared__ __align__(8) uint64_t s_bar[2];
    __shared__ Rec s_bnd[5]; // A[a0-1], A[a1], B[b0-1], B[b1], the tile's last record
    __shared__ unsigned long long s_wb[NT / 32];
    __shared__ uint32_t s_wc[NT / 32];
    __shared__ unsigned long long s_pref[2];
    __shared__ uint32_t s_rbase[kFinMaxRunsSmem + 1];
    __shared__ uint8_t s_rlut[256]; // run that holds gid (b << lut_shift): a record's run is that one or a close successor
    __shared__ const uint4 *s_rindex[kFinMaxRunsSmem];
    __shared__ const uint8_t *s_rdata[kFinMaxRunsSmem];

    pdl_trigger();
    pdl_wait();
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t skip = p.ctl->prefix_len + kWindowBytes;
    const uint32_t n_tiles = p.tile_base[level][p.nseg[level + 1]];
    const uint32_t G = gridDim.x;
    uint32_t tile = blockIdx.x;
    if (tile >= n_tiles) return;
    const bool runs_cached = p.n_runs <= (uint32_t)kFinMaxRunsSmem;
    uint32_t lut_shift = 0;
    while (((uint64_t)p.n_total >> lut_shift) > 256) lut_shift++; // gid >> lut_shift < 256 for every gid < n_total
    if (runs_cached) {
        for (uint32_t r = tid; r < p.n_runs; r += NT) {
            s_rbase[r] = p.runs[r].base;
            s_rindex[r] = p.runs[r].index;
            s_rdata[r] = p.runs[r].data;
        }
        if (tid == 0) s_rbase[p.n_runs] = 0xFFFFFFFFu; // sentinel: no run starts above any gid
        s_rlut[tid] = (uint8_t)find_run(p, (uint32_t)(((uint64_t)tid << lut_shift) < p.n_total ? (uint64_t)tid << lut_shift : p.n_total - 1));
    }
    if (tid == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        s_pref[0] = s_pref[1] = ~0ull; // tag 0xFFFF: no tile's
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    FIN_PH_DECL

    // entry address / key_size / full_size of the entry behind a gid: its run's index record (64-byte granule)
    auto run_of = [&](uint32_t gid) -> uint32_t {
        if (!runs_cached) return find_run(p, gid);
        uint32_t r = s_rlut[gid >> lut_shift]; // owner of the bucket's first gid; ours is the last run whose base <= gid
        while (s_rbase[r + 1] <= gid) r++;
        return r;
    };
    auto index_ptr = [&](uint32_t gid, uint32_t r) -> const uint4 * {
        return runs_cached ? s_rindex[r] + (gid - s_rbase[r]) : p.runs[r].index + (gid - p.runs[r].base);
    };
    auto data_ptr = [&](uint32_t r) -> const uint8_t * { return runs_cached ? s_rdata[r] : p.runs[r].data; };

    auto issue = [&](const FinDesc &d, Rec *buf, uint64_t *bar) { // thread 0 only
        const uint32_t ap = d.nb & 1u, an = (d.nb >> 1) & 1u, bp = (d.nb >> 2) & 1u, bn = (d.nb >> 3) & 1u;
        const uint32_t ca = d.n_a + ap + an, cb = d.n_b + bp + bn;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // the buffer was last written through the generic proxy
        mbar_expect_tx(bar, (ca + cb) * 16u);
        if (ca) tma_load_1d(buf + 1 - ap, &src[d.a_src - ap], ca * 16u, bar);
        if (cb) tma_load_1d(buf + d.n_a + 3 - bp, &src[d.b_src - bp], cb * 16u, bar);
    };

    // Tile descriptors from k_merge_partition's boundary records (already moved past straddling groups): the boundary index
    // three tiles ahead, the two records two tiles ahead -- no dependent chain inside an iteration.  The last level of a
    // single compaction is one pair: segments 0 (A) and 1 (B).
    const Seg segA = p.seg[level][0];
    Seg segB;
    segB.start = 0; segB.len = 0;
    if (p.nseg[level] > 1) segB = p.seg[level][1];
    auto ld_bidx = [&](uint32_t t) -> uint32_t { return t < n_tiles ? __ldg(&p.tile_bnd[t]) : 0xFFFFFFFFu; };
    auto mk_desc = [&](uint32_t bidx) -> FinDesc {
        FinDesc d;
        d.a_src = d.n_a = d.b_src = d.n_b = d.a_end = d.b_end = d.diag0 = d.nb = 0;
        if (bidx == 0xFFFFFFFFu) return d;
        const uint4 b0 = __ldg(&p.bnd[bidx]), b1 = __ldg(&p.bnd[bidx + 1]);
        d.a_src = b0.x; d.n_a = b1.x - b0.x;
        d.b_src = b0.y; d.n_b = b1.y - b0.y;
        d.a_end = segA.start + segA.len;
        d.b_end = segB.start + segB.len;
        d.diag0 = b0.z;
        d.nb = (b0.x > segA.start ? 1u : 0u) | (b1.x < d.a_end ? 2u : 0u) | (b0.y > segB.start ? 4u : 0u) | (b1.y < d.b_end ? 8u : 0u);
        return d;
    };
    FinDesc cur = mk_desc(ld_bidx(tile));
    FinDesc nxt = mk_desc(ld_bidx(tile + G));
    uint32_t bidx2 = ld_bidx(tile + 2 * G);
    if (tid == 0) issue(cur, bufs[0], &s_bar[0]);
    const int keep_tombstones = p.keep_tombstones;

    // One-tile software pipeline: tile q publishes its aggregate as soon as it is resolved, and its look-back and emit run in
    // the next iteration, after tile q+1 has been merged and its index loads are in flight (or after the loop, for the CTA's
    // last tile).  By then the tiles before q have had one iteration to publish, so the look-back rarely waits.
    // Why a tile never waits on a CTA that is waiting on it: the look-back of tile t waits only for tiles < t to publish their
    // aggregates, and a CTA publishes the aggregate of its tile t after running only the look-backs of its own earlier tiles
    // (all < t) and nothing that waits on a later tile.  By induction on t every aggregate gets published, given that every
    // CTA holding a tile is resident -- the same co-residency as a non-pipelined chained scan, which the grid is sized for
    // at engine creation.
    // Tile q's survivors wait in s_tlo / s_thi (entry address / {key_size, full_size}), free between the last head of q and
    // the timestamp stores of q+1.  A thread keeps its survivors in the very slots it later stores its own timestamps to
    // (d + i, d = 7 * tid whenever it has records), so neither the emit nor those stores need a CTA barrier -- a barrier
    // would wait for the timestamp loads in flight.  The look-back's result reaches the other warps the same way, through
    // two shared words that each carry the tile's tag.
    uint32_t prev_tile = 0, prev_d = 0, prev_act = 0, prev_pos = 0, prev_tc = 0;
    unsigned long long prev_off = 0, prev_tb = 0;
    volatile unsigned long long *vpref = s_pref; // {tag << 48 | bytes before the tile (< 2^48), tag << 32 | entries before it}
    auto finish_prev = [&](uint32_t prev_q) {
        const unsigned long long tag = prev_q & 0xFFFFu; // differs from the previous tile's (and from the initial 0xFFFF at q = 0)
        if (warp == 0) { // the look-back is one warp's: 128 predecessors per step, stops at the nearest inclusive prefix
            unsigned long long eb = 0;
            uint32_t ec = 0;
            if (prev_tile > 0) fin_lookback(p.scan_state, prev_tile, lane, eb, ec);
            if (lane == 0) {
                if (prev_tile > 0) {
                    unsigned long long *mine = p.scan_state + 2ull * prev_tile;
                    st_volatile_u64(mine, (kScanPrefix << 62) | (eb + prev_tb));
                    st_volatile_u64(mine + 1, (kScanPrefix << 32) | (unsigned long long)(ec + prev_tc));
                }
                vpref[0] = (tag << 48) | eb;
                vpref[1] = (tag << 32) | ec;
                if (prev_tile + 1 == n_tiles) { // the last tile holds the totals
                    Ctl *cw = p.ctl;
                    cw->out_data_len = eb + prev_tb;
                    cw->out_items = ec + prev_tc;
                }
            }
        }
        unsigned long long pb, pc;
        do {
            pb = vpref[0];
            pc = vpref[1];
        } while ((pb >> 48) != tag || (pc >> 32) != tag);
        FIN_PH(4);
        // ---- emit: .index records (entry_writer.rs:76-86), source addresses, gather-tile markers
        unsigned long long off = (pb & ((1ull << 48) - 1)) + prev_off; // within this job's .data
        uint32_t pos = (uint32_t)pc + prev_pos;
        constexpr unsigned long long gt = kGatherTileBytes;
#pragma unroll
        for (int i = 0; i < VT; i++) {
            if (!((prev_act >> i) & 1u)) continue;
            const unsigned long long sz = s_thi[prev_d + i];
            const uint32_t fs = (uint32_t)(sz >> 32);
            if (!fs) continue;
            const unsigned long long file_off = off + p.out_offset_base;
            p.out_index[pos] = make_uint4((uint32_t)file_off, (uint32_t)(file_off >> 32), (uint32_t)sz, fs);
            p.src_ptr[pos] = s_tlo[prev_d + i];
            for (unsigned long long bq = (off + gt - 1) / gt; bq * gt < off + fs && bq < p.tile_first_n; bq++) p.tile_first[bq] = pos;
            off += fs;
            pos++;
        }
        FIN_PH(5);
    };

    uint32_t q = 0;
    for (;; q++) {
        Rec *s = bufs[q & 1];
        uint4 *s4 = reinterpret_cast<uint4 *>(s);
        const bool has_next = tile + G < n_tiles;
        if (tid == 0 && has_next) issue(nxt, bufs[(q + 1) & 1], &s_bar[(q + 1) & 1]);
        const FinDesc nn = mk_desc(bidx2);            // consumed one iteration from now
        const uint32_t bidx3 = ld_bidx(tile + 3 * G); // ... and two iterations from now
        while (!mbar_try_wait(&s_bar[q & 1], (q >> 1) & 1)) {}
        FIN_PH(0);

        // ---- merge-path: thread t produces merged records [7t, 7t + 7) of the tile
        const uint32_t nA = cur.n_a, nB = cur.n_b, n = nA + nB;
        const Rec *A = s + 1, *B = s + nA + 3;
        uint32_t d = tid * VT;
        if (d > n) d = n;
        Rec me[VT + 1]; // this thread's merged records, then the one after them
        {
            uint32_t lo = d > nB ? d - nB : 0;
            uint32_t hi = d < nA ? d : nA;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (!key_less_smem(p, skip, &B[d - 1 - mid], &A[mid])) lo = mid + 1; else hi = mid;
            }
            uint32_t ai = lo, bi = d - lo;
            Rec ak = A[ai], bk = B[bi]; // may read one slot past a range: the neighbour slots
#pragma unroll
            for (int i = 0; i < VT; i++) {
                const bool has_a = ai < nA, has_b = bi < nB;
                const bool take_b = has_b && (!has_a || key_less(p, skip, bk, ak));
                me[i] = take_b ? bk : ak;
                if (take_b) { bi++; bk = B[bi]; } else { ai++; ak = A[ai]; }
            }
            if (tid == 0) {
                s_bnd[0] = s[0];
                s_bnd[1] = s[nA + 1];
                s_bnd[2] = s[nA + 2];
                s_bnd[3] = s[nA + 3 + nB];
            }
            __syncthreads(); // every thread is done reading the unmerged ranges
            // only a thread's first and last record are ever read by its neighbours (group flags across thread borders)
            if (d < n) s[d] = me[0];
            if (d + VT - 1 < n) s[d + VT - 1] = me[VT - 1];
#pragma unroll
            for (int i = 0; i < VT; i++)
                if (d + i == n - 1) s_bnd[4] = me[i];
        }
        __syncthreads();
        FIN_PH(1);

        // ---- resolve, part 1: group flags from the neighbours' keys, index record of every entry
        uint32_t m_act = 0, m_eqn = 0, m_eqp = 0;
        uint32_t gidv[VT];
        uint4 irec[VT];
        {
#pragma unroll
            for (int i = 0; i < VT; i++)
                if (d + i < n) m_act |= 1u << i;
            me[VT].x = me[VT].y = me[VT].z = me[VT].w = 0;
            if (d + VT < n) me[VT] = s[d + VT];
#pragma unroll
            for (int i = 0; i < VT; i++) {
                if (!(m_act & (1u << i))) continue;
                bool eqn;
                if (d + i + 1 < n) {
                    eqn = key_equal(p, skip, me[i], me[i + 1]);
                } else { // the tile's last record: the next merged record is A[a1] or B[b1]
                    eqn = ((cur.nb & 2u) && key_equal(p, skip, me[i], s_bnd[1])) || ((cur.nb & 8u) && key_equal(p, skip, me[i], s_bnd[3]));
                }
                if (eqn) m_eqn |= 1u << i;
            }
            m_eqp = m_eqn << 1;
            if (m_act & 1u) {
                bool eqp;
                if (d > 0) eqp = key_equal(p, skip, s[d - 1], me[0]);
                else eqp = ((cur.nb & 1u) && key_equal(p, skip, s_bnd[0], me[0])) || ((cur.nb & 4u) && key_equal(p, skip, s_bnd[2], me[0]));
                if (eqp) m_eqp |= 1u;
            }
#pragma unroll
            for (int i = 0; i < VT; i++) {
                gidv[i] = me[i].w;
                irec[i] = make_uint4(0, 0, 0, 0);
                if (m_act & (1u << i)) {
                    const uint32_t r = run_of(gidv[i]);
                    const uint4 *q4 = index_ptr(gidv[i], r);
                    irec[i] = kNarrow ? ldg128_narrow(q4) : __ldg(q4);
                }
            }
        }
        __syncthreads(); // every neighbour key has been read: the tile's slots may now hold {entry address, key_size, full_size}
        FIN_PH(2);
        {
            const uint32_t m_grp = m_act & (m_eqn | m_eqp); // members of a group of two or more
            unsigned long long tlo[VT], thi[VT];
#pragma unroll
            for (int i = 0; i < VT; i++) {
                tlo[i] = thi[i] = 0;
                if (!(m_act & (1u << i))) continue;
                const uint32_t r = run_of(gidv[i]);
                const uint8_t *entry = data_ptr(r) + ((uint64_t)irec[i].x | ((uint64_t)irec[i].y << 32));
                const unsigned long long ea = (unsigned long long)(uintptr_t)entry;
                // {entry address, key_size, full_size} of position d + i; in shared memory, not registers, across the emit below
                s4[d + i] = make_uint4((uint32_t)ea, (uint32_t)(ea >> 32), irec[i].z, irec[i].w);
                if ((m_grp >> i) & 1u) { // its timestamp decides (mod.rs:80)
                    const uint8_t *t = entry + irec[i].w - 16;
                    if (kNarrow) { tlo[i] = ld_u64_unaligned_narrow(t); thi[i] = ld_u64_unaligned_narrow(t + 8); }
                    else { tlo[i] = ld_u64_unaligned(t); thi[i] = ld_u64_unaligned(t + 8); }
                    s_flag[d + i] = (uint8_t)((m_eqn >> i) & 1u);
                }
            }
            FIN_PH(3);
            // the previous tile's look-back and emit while this tile's timestamps travel: no CTA barrier until they are stored
            if (q > 0) finish_prev(q - 1);
#pragma unroll
            for (int i = 0; i < VT; i++) {
                if ((m_grp >> i) & 1u) { s_tlo[d + i] = tlo[i]; s_thi[d + i] = thi[i]; }
            }
        }
        __syncthreads();
        FIN_PH(6);

        // ---- resolve, part 2: heads pick their group's winner; the tombstone rule (lsm_tree.rs:1045-1046)
        unsigned long long vb = 0;
        uint32_t vc = 0;
        uint4 we[VT]; // what is written for position d + i: {entry address, key_size, full_size or 0}
#pragma unroll
        for (int i = 0; i < VT; i++) {
            we[i] = make_uint4(0, 0, 0, 0);
            if (!((m_act >> i) & 1u) || ((m_eqp >> i) & 1u)) continue; // not a head
            const uint32_t k = d + i;
            uint4 info = s4[k];
            if ((m_eqn >> i) & 1u) {
                unsigned long long wlo = s_tlo[k], whi = s_thi[k];
                uint32_t j = k;
                bool more = true;
                while (more && j + 1 < n) { // members inside the tile, in run-position order: a later member wins ties
                    j++;
                    const unsigned long long clo = s_tlo[j], chi = s_thi[j];
                    if (!ts_greater(wlo, whi, clo, chi)) { info = s4[j]; wlo = clo; whi = chi; }
                    more = s_flag[j] != 0;
                }
                if (more) {
                    // The group runs past the tile: its remaining members are the records of A from a1 on and then of B from
                    // b1 on that carry the same key -- still in run-position order (a group that continues in A has no member
                    // from B inside the tile: ties take A first).
                    const Rec last = s_bnd[4];
                    for (int side = 0; side < 2; side++) {
                        uint32_t g = side ? cur.b_src + nB : cur.a_src + nA;
                        const uint32_t end = side ? cur.b_end : cur.a_end;
                        for (; g < end; g++) {
                            const Rec nx = ld_rec(&src[g]);
                            if (!key_equal(p, skip, last, nx)) break;
                            const KeyRef ck = key_of_gid(p, nx.w);
                            uint64_t clo, chi;
                            ld_ts(ck.entry, ck.full_size, &clo, &chi);
                            if (!ts_greater(wlo, whi, clo, chi)) {
                                const unsigned long long ea = (unsigned long long)(uintptr_t)ck.entry;
                                info = make_uint4((uint32_t)ea, (uint32_t)(ea >> 32), ck.klen + 8, ck.full_size);
                                wlo = clo; whi = chi;
                            }
                        }
                    }
                }
            }
            const bool tomb = info.w == info.z + 24;
            if (keep_tombstones || !tomb) {
                we[i] = info;
                vb += info.w;
                vc += 1;
            }
        }

        // ---- scan: this thread's survivors -> tile -> all tiles before this one
        unsigned long long ib = vb;
        uint32_t ic = vc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long xb = __shfl_up_sync(0xFFFFFFFFu, ib, o);
            const uint32_t xc = __shfl_up_sync(0xFFFFFFFFu, ic, o);
            if (lane >= (uint32_t)o) { ib += xb; ic += xc; }
        }
        if (lane == 31) { s_wb[warp] = ib; s_wc[warp] = ic; }
        __syncthreads(); // every head is done with s_tlo / s_thi / s4
        unsigned long long tb = 0, wbefore = 0;
        uint32_t tc = 0, wcbefore = 0;
#pragma unroll
        for (int w = 0; w < NT / 32; w++) {
            if ((uint32_t)w < warp) { wbefore += s_wb[w]; wcbefore += s_wc[w]; }
            tb += s_wb[w];
            tc += s_wc[w];
        }
        if (tid == 0) { // tile 0's aggregate is its inclusive prefix; no other tile waits for anything before publishing
            // Each word says what it holds (aggregate or inclusive prefix): a reader needs both words at the same stage and
            // simply reads again when it caught the pair mid-update -- no fence on either side.
            const unsigned long long st = tile == 0 ? kScanPrefix : kScanAgg;
            unsigned long long *mine = p.scan_state + 2ull * tile;
            st_volatile_u64(mine, (st << 62) | tb);
            st_volatile_u64(mine + 1, (st << 32) | tc);
        }
#pragma unroll
        for (int i = 0; i < VT; i++) {
            if ((m_act >> i) & 1u) {
                s_tlo[d + i] = (unsigned long long)we[i].x | ((unsigned long long)we[i].y << 32);
                s_thi[d + i] = (unsigned long long)we[i].z | ((unsigned long long)we[i].w << 32);
            }
        }
        prev_tile = tile;
        prev_d = d;
        prev_act = m_act;
        prev_off = wbefore + ib - vb;
        prev_pos = wcbefore + ic - vc;
        prev_tb = tb;
        prev_tc = tc;
        if (!has_next) {
            FIN_PH(7);
            break;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // generic-proxy accesses of this buffer before the next bulk copy into it
        __syncthreads(); // s_bnd / the tile buffer are free for the next tile
        FIN_PH(7);
        tile += G;
        cur = nxt;
        nxt = nn;
        bidx2 = bidx3;
    }
    finish_prev(q);
#ifdef DBEEL_FIN_PHASES
    if (tid == 0) fin_phase_flush(ph_acc, n_tiles);
#endif
}

} // namespace dbeel
