// gather_h.cuh -- K5 at Hopper's access width (k_gather_h, DBEEL_GATHER=11, the default).
//
// k_gather32 was built around single 256-bit global accesses, which sm_90 does not have: there every 32-byte lane
// granule is two 128-bit accesses 32 bytes apart, so one warp instruction spans 1 KB in 16-byte pieces.  This kernel
// keeps k_gather32's skeleton -- short-lived CTAs, one 8 KB output tile each, one barrier after the metadata staging,
// the payload held in registers, the OR-reduce + popcount vector -> entry map, a dense one-lane-per-entry boundary
// pass, the filter as the epilogue -- and changes what the H100 does differently:
//   * 16-byte output vectors, lane-contiguous (k_gather's mapping): a warp store covers 512 contiguous bytes, a warp
//     load at most 528 contiguous source bytes of one entry.  The second aligned source vector is loaded only when the
//     source shift is nonzero.
//   * The boundary vector (the one holding entry j's last byte) gets its tail and its head from only the aligned 16-byte
//     chunks that hold wanted bytes (chunks16), blended in registers (blend16), one 16-byte store.
//   * The filter's REDs carry an L2 evict_last policy (kernels.cuh), so the ~4 GB payload stream does not push filter
//     sectors out of the 50 MB L2 between two touches.  Marking the payload evict_first as well did not pay (DESIGN.md §7).
// Same Params contract as k_gather32 (hash_rec, bloom_elsewhere, out_offset_base, multi-megabyte entries, no filter);
// output buffers 16-byte aligned, which every entry point checks.
#pragma once
#include "kernels.cuh"

namespace dbeel {

#ifndef DBEEL_GATHER_H_VPT
#define DBEEL_GATHER_H_VPT 4 // 16-byte output vectors per thread: 64 bytes of payload in flight, as k_gather32
#endif
constexpr int kGhVpt = DBEEL_GATHER_H_VPT;
constexpr int kGhThreads = (int)(kGatherTileBytes / (16ull * 32 * kGhVpt)) * 32; // one 8 KB tile per CTA
static_assert(kGatherTileBytes == 16ull * kGhThreads * kGhVpt, "gather tile = 16 bytes x threads x vectors");
#ifndef DBEEL_GATHER_H_MINB
#define DBEEL_GATHER_H_MINB (1024 / kGhThreads) // 8 CTAs of 128 threads: 64 registers, no spills
#endif

// 16 bytes at an arbitrary address of which bytes [lo, hi) are wanted: only the aligned chunks that hold them are loaded
__device__ __forceinline__ uint4 ld16_lean(uintptr_t a, uint32_t lo, uint32_t hi) {
    const uint32_t s0 = (uint32_t)(a & 15);
    const uint4 *sv = reinterpret_cast<const uint4 *>(a - s0);
    const uint32_t m = chunks16(s0, lo, hi);
    uint4 X = make_uint4(0, 0, 0, 0), Y = make_uint4(0, 0, 0, 0);
    if (m & 1u) X = __ldg(sv);
    if (m & 2u) Y = __ldg(sv + 1);
    return realign16_sel(X, Y, s0);
}

__global__ void __launch_bounds__(kGhThreads, DBEEL_GATHER_H_MINB) k_gather_h(Params p) {
    pdl_trigger();
    pdl_wait();
    constexpr int NT = kGhThreads;
    constexpr int VPT = kGhVpt;
    __shared__ unsigned long long s_adj[kGatherMaxEntries]; // entry address minus its tile-relative start
    __shared__ int s_r0[kGatherMaxEntries], s_r1[kGatherMaxEntries];
    __shared__ uint32_t s_ks[kGatherMaxEntries];
    const Ctl *c = p.ctl;
    const unsigned long long out_len = c->out_data_len;
    // A caller's payload bound that turns out too low (sparse batches) is only reported after the job: the grid was sized
    // from the bound, so the tiles stop writing there and entries keep their places in the true stream (out_len).
    const unsigned long long out_end = out_len < p.data_bound ? out_len : p.data_bound;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile_id = blockIdx.x;
    const unsigned long long T0 = (unsigned long long)tile_id * kGatherTileBytes;
    if (T0 >= out_end) return;
    const uint32_t tile_len = out_end - T0 < kGatherTileBytes ? (uint32_t)(out_end - T0) : (uint32_t)kGatherTileBytes;
    const uint32_t e_lo = p.tile_first[tile_id];
    const uint32_t e_hi = T0 + kGatherTileBytes < out_len ? p.tile_first[tile_id + 1] : c->out_items - 1;
    const uint32_t ne = e_hi - e_lo + 1; // <= kGatherMaxEntries: every entry is >= 32 bytes
    const bool hash_here = p.bloom.words != nullptr && p.hash_rec == nullptr && !p.bloom_elsewhere;
    for (uint32_t j = tid; j < ne; j += NT) {
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

    // ---- copy: warp w owns bytes [w * 512 VPT, (w + 1) * 512 VPT) of the tile, 512 bytes (32 lanes x 16) at a time
    uint4 *dst_tile = reinterpret_cast<uint4 *>(p.out_data + T0);
    const int sub0 = (int)(warp * (uint32_t)(512 * VPT));
    if ((uint32_t)sub0 < tile_len) {
        uint32_t j = 0; // the entry that holds byte sub0 = number of entries ending at or before it (ends ascend)
        for (uint32_t base = 0; base + 1 < ne; base += 32) {
            const uint32_t i = base + lane;
            j += __popc(__ballot_sync(0xFFFFFFFFu, i + 1 < ne && s_r1[i] <= sub0));
        }
        uint4 A[VPT], B[VPT];
        uint32_t sh[VPT];
        bool pure[VPT];
        const uint32_t lanes_le = 0xFFFFFFFFu >> (31 - lane); // bits 0..lane
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            const int cb = sub0 + k * 512;
            const int b0 = cb + (int)lane * 16;
            // Entries that end inside the chunk, i.e. in (cb, cb + 512]: at most 17 (entries are >= 32 bytes), lane l looks
            // at entry j + l.  An end at r1 precedes the vectors t = ceil((r1 - cb) / 16) .. 31; distinct entries, distinct t.
            const uint32_t i = j + lane;
            const int r1 = i + 1 < ne ? s_r1[i] : 0x7FFFFFFF;
            const bool ends_here = r1 <= cb + 512;
            const uint32_t t = (uint32_t)((ends_here ? r1 : cb + 16) - cb + 15) >> 4; // 1..32 when ends_here
            const uint32_t ends = __reduce_or_sync(0xFFFFFFFFu, (ends_here && t < 32) ? (1u << t) : 0u);
            const uint32_t cnt = __popc(ends & lanes_le); // entries ending at or before my vector's first byte
            const uint32_t adv = __popc(__ballot_sync(0xFFFFFFFFu, ends_here));
            const uint32_t e = j + cnt; // entry that holds byte b0
            j += adv;                   // entry that holds the next chunk's first byte
            // Unconditional loads: a vector that is not wholly inside entry e (it holds e's end, or lies past the end of the
            // stream) reads the last 16 bytes of e instead (always valid: entries are >= 32 bytes) and is not stored here.
            const int r1e = s_r1[e];
            pure[k] = (uint32_t)b0 + 16 <= tile_len && b0 + 16 <= r1e;
            const int bl = b0 + 16 <= r1e ? b0 : r1e - 16;
            const uintptr_t sa = (uintptr_t)(s_adj[e] + (unsigned long long)(long long)bl);
            sh[k] = (uint32_t)(sa & 15);
            const uint4 *sv = reinterpret_cast<const uint4 *>(sa - sh[k]);
            A[k] = __ldg(sv);
            B[k] = A[k];
            if (sh[k]) B[k] = __ldg(sv + 1);
        }
#pragma unroll
        for (int k = 0; k < VPT; k++) {
            if (pure[k]) dst_tile[(uint32_t)(sub0 >> 4) + (uint32_t)k * 32 + lane] = realign16_sel(A[k], B[k], sh[k]);
        }
    }

    // ---- the vector that holds the last byte of entry j (unless j ends on a vector boundary): tail of j, head of j + 1
    for (uint32_t j = tid; j < ne; j += NT) {
        const int r1 = s_r1[j];
        if (r1 <= 0 || (r1 & 15) == 0 || r1 > (int)tile_len) continue;
        const uint32_t b0 = (uint32_t)r1 & ~15u, t = (uint32_t)r1 - b0; // t = 1..15 bytes of entry j in this vector
        const uint4 T = ld16_lean((uintptr_t)(s_adj[j] + b0), 0u, t);
        if (b0 + 16u <= tile_len) { // the rest of the vector is the head of entry j + 1 (entries are >= 32 bytes)
            const uint4 H = ld16_lean((uintptr_t)(s_adj[j + 1] + b0), t, 16u);
            const uint32_t tw[4] = {T.x, T.y, T.z, T.w}, hw[4] = {H.x, H.y, H.z, H.w};
            uint32_t o[4];
            blend16(tw, hw, t, o);
            dst_tile[b0 >> 4] = make_uint4(o[0], o[1], o[2], o[3]);
        } else { // ragged end of the whole stream: never write past out_data_len
            const uint32_t tw[4] = {T.x, T.y, T.z, T.w};
            uint8_t *d = p.out_data + T0;
            for (uint32_t b = 0; b < t; b++) d[b0 + b] = (uint8_t)(tw[b >> 2] >> ((b & 3) * 8));
        }
    }

    // ---- bloom (fused epilogue), only when k_extract did not hash: entries whose first byte lies in this tile
    if (hash_here) {
        const uint64_t keep = l2_evict_last();
        for (uint32_t j = tid; j < ne; j += NT) {
            const int r0 = s_r0[j];
            if (r0 < 0 || r0 >= (int)kGatherTileBytes) continue;
            const uint8_t *key = reinterpret_cast<const uint8_t *>((uintptr_t)(s_adj[j] + (unsigned long long)r0)) + 8;
            const uint64_t klen = s_ks[j] - 8;
            uint64_t h0, h1;
            sip13_pair_vec_u8(p.bloom.sip, klen, [key](uint64_t q) { return ld_u64_unaligned(key + 8 * q); }, &h0, &h1);
            uint32_t *words = p.bloom.words;
            bloom_probe_all(h0, h1, p.bloom.k_num, p.bloom.bits, p.bloom.bits_magic,
                            [words, keep](uint64_t bit) { red_or_keep(&words[bit >> 5], 1u << (bit & 31), keep); });
        }
    }
}

} // namespace dbeel
