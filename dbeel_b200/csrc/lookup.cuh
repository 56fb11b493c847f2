// lookup.cuh -- row N2 of the scope table: the read side of the files the compaction path writes.
//
// get_entry's SSTable loop (lsm_tree.rs:686-719): newest table first, `bloom.check(key)` (:692-696)
// rules a table out, otherwise `binary_search` (:605-670) probes the .index / .data pair.  One
// thread per query key; tens of thousands of keys in flight hide the dependent probe chain
// (index record -> entry key -> compare), and the upper levels of every search stay L2-resident.
//
// Two search modes:
//   DBEEL_LOOKUP_REFERENCE  the reference's loop restated step for step, including its exit right
//                           after index 0 has been probed (`half == 0`, :660) -- some present keys
//                           are reported absent, exactly as the reference reports them
//                           (oracle: orc_sstable_lookup; tests/test_oracle_goldens.py);
//   DBEEL_LOOKUP_EXACT      a plain lower-bound search that finds every key that is present.
//
// k_lookup writes the rows (dbeel_get_many*); k_lookup_emit runs the same search and also hands each query's entry to the
// scan's split and phase 2 (dbeel_get_values*: the entries come back as one arrival batch in query order).
#pragma once

#include "kernels.cuh"
#include "scan.cuh"

namespace dbeel {

struct TableDesc {
    const uint8_t *data;
    uint64_t data_len;
    const uint4 *index;
    uint64_t n;            // entries = len(.index) / 16 (lsm_tree.rs:452-453)
    const uint32_t *words; // bloom bit vector inside the .bloom file, or null (no filter: lsm_tree.rs:94-101)
    uint64_t bits, bits_magic;
    uint32_t k_num, pad;
    uint64_t sip[4];
};

struct LookupParams {
    const TableDesc *tables;
    uint32_t n_tables;
    uint32_t mode;
    const uint8_t *keys;     // query keys back to back
    const uint64_t *key_off; // n_keys + 1 offsets into `keys`
    uint64_t n_keys;
    uint4 *out;              // dbeel_lookup_result rows
};

// `nbytes` (1..8) bytes at p as a little-endian integer (upper bytes unspecified).  Touches only the aligned 8-byte
// words that hold requested bytes, so a key that ends at the last byte of its buffer is never over-read.
template <bool kNarrow>
__device__ __forceinline__ uint64_t ld_bytes_le(const uint8_t *p, uint32_t nbytes) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t mis = (uint32_t)(a & 7);
    const uint64_t *w = reinterpret_cast<const uint64_t *>(a - mis);
    uint64_t v = (kNarrow ? ldg64_narrow(w) : __ldg(w)) >> (8 * mis);
    if (mis + nbytes > 8) v |= (kNarrow ? ldg64_narrow(w + 1) : __ldg(w + 1)) << (64 - 8 * mis);
    return v;
}

// Ordering of `Vec<u8>::cmp` (lsm_tree.rs:636): bytes, then length.  <0, 0, >0 like memcmp.
// a = key bytes inside an SSTable (random access: 64-byte L2 granules), b = the query key.
__device__ __forceinline__ int cmp_key_bytes(const uint8_t *a, uint64_t alen, const uint8_t *b, uint64_t blen) {
    const uint64_t m = alen < blen ? alen : blen;
    for (uint64_t o = 0; o < m; o += 8) {
        const uint32_t nb = m - o < 8 ? (uint32_t)(m - o) : 8u;
        uint64_t x = ld_bytes_le<true>(a + o, nb), y = ld_bytes_le<false>(b + o, nb);
        if (nb < 8) {
            const uint64_t mask = ~0ull >> (8 * (8 - nb));
            x &= mask;
            y &= mask;
        }
        if (x != y) { // first differing byte decides: compare big-endian
            const uint64_t xs = __byte_perm((uint32_t)(x >> 32), 0, 0x0123) | ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32);
            const uint64_t ys = __byte_perm((uint32_t)(y >> 32), 0, 0x0123) | ((uint64_t)__byte_perm((uint32_t)y, 0, 0x0123) << 32);
            return xs < ys ? -1 : 1;
        }
    }
    return alen < blen ? -1 : (alen > blen ? 1 : 0);
}

constexpr uint32_t kLookupCorrupt = 0x80000000u;  // an index record pointed outside its .data file
constexpr uint32_t kLookupBadEntry = 0x40000000u; // k_lookup_emit: the hit's entry does not decode (get_entry returns Err)

// compare the key of entry `rec` of table t with the query: sets *bad when the record cannot be decoded; *ix_out = the index
// record (the emitting form decodes a hit's entry from it without loading it again)
__device__ __forceinline__ int probe(const TableDesc &t, uint64_t rec, const uint8_t *key, uint64_t klen, bool *bad, uint4 *ix_out) {
    const uint4 ix = ldg128_narrow(&t.index[rec]);
    *ix_out = ix;
    const uint64_t off = (uint64_t)ix.x | ((uint64_t)ix.y << 32);
    if (off > t.data_len || t.data_len - off < 8) { *bad = true; return 0; }
    const uint64_t cur_klen = ld_bytes_le<true>(t.data + off, 8); // bincode Vec<u8>: u64 length, then the bytes
    if (cur_klen > t.data_len - off - 8) { *bad = true; return 0; }
    return cmp_key_bytes(t.data + off + 8, cur_klen, key, klen);
}

#ifndef DBEEL_LOOKUP_MINB
#define DBEEL_LOOKUP_MINB 4 // 4 CTAs of 256 threads per SM = a 64-register cap
#endif
// dbeel_get_values*: per query the destination of its entry (0 = answered, kScanNone = no entry) and the 16-byte record
// {source address, 8 + klen, full_size} the scan's phase 2 splits and gathers (scan.cuh)
struct LookupEmit {
    uint32_t *dest;
    uint4 *flat;
};

// The search of one query key, shared by k_lookup (rows only) and k_lookup_emit (rows + the hit's entry as a split record).
// kEmit decodes the hit the way binary_search does after the key compared equal (lsm_tree.rs:628-651): the key frame
// read_at(offset, key_size) must be exactly the key (bincode reject_trailing_bytes: key_size == 8 + klen), and
// read_at(offset + key_size, full_size - key_size) exactly one EntryValue (u64 dlen | data | i128 ts inside `time`'s
// range) inside .data.  A hit that does not decode gets kLookupBadEntry and no entry: the reference's `?` returns Err
// there, so no older table is tried either.
template <bool kEmit>
__device__ __forceinline__ void lookup_query(const LookupParams &p, const LookupEmit &em) {
    const uint64_t q = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    if (q >= p.n_keys) return;
    const uint64_t k0 = p.key_off[q];
    const uint8_t *key = p.keys + k0;
    const uint64_t klen = p.key_off[q + 1] - k0;
    int32_t found_table = -1;
    uint32_t rejects = 0;
    uint64_t record = 0;
    uint4 hit_ix = make_uint4(0, 0, 0, 0);
    for (uint32_t ti = p.n_tables; ti-- > 0 && found_table < 0;) { // sstables.iter().rev(): newest first (:688)
        const TableDesc &t = p.tables[ti];
        if (t.words != nullptr) { // :691-696
            uint64_t h0, h1;
            sip13_pair_vec_u8(t.sip, klen, [key, klen](uint64_t w) {
                const uint64_t left = klen - 8 * w;
                return ld_bytes_le<false>(key + 8 * w, left < 8 ? (uint32_t)left : 8u); // the tail is masked by the caller
            }, &h0, &h1);
            bool all = true;
            const uint32_t *words = t.words;
            bloom_probe_all(h0, h1, t.k_num, t.bits, t.bits_magic,
                            [&all, words](uint64_t bit) { all = all && ((__ldg(&words[bit >> 5]) >> (bit & 31)) & 1u); });
            if (!all) { rejects++; continue; }
        }
        const uint64_t n = t.n;
        if (n == 0) continue;
        bool bad = false;
        if (p.mode == 0) { // the reference's loop, :612-667
            // Written with one exit test and selects instead of the reference's five `break`s: with early exits the
            // compiler keeps lanes that left the comparison on different sides apart until the search ends (no
            // reconvergence point inside the loop), which ran the warp's 32 searches almost one after another.
            uint64_t half = n / 2, high = n - 1, low = 0;
            bool done = false;
            while (!done) {
                uint4 ix;
                const int c = probe(t, half, key, klen, &bad, &ix);
                const bool hit = c == 0 && !bad;
                if (hit) { found_table = (int32_t)ti; record = half; hit_ix = ix; }
                low = c < 0 ? half + 1 : low;                              // Ordering::Less
                high = c > 0 ? (half > 1 ? half : 1) - 1 : high;           // Ordering::Greater: max(half, 1) - 1
                done = hit || bad || half == 0 || half == n;               // `if half == 0 || half == length { break }`
                half = (high + low) / 2;
                done = done || low > high;                                 // `while not: low_index > high_index`
            }
        } else { // every present key is found
            uint64_t lo = 0, hi = n;
            while (lo < hi && !bad) {
                const uint64_t mid = lo + (hi - lo) / 2;
                uint4 ix;
                const int c = probe(t, mid, key, klen, &bad, &ix);
                if (c == 0 && !bad) { found_table = (int32_t)ti; record = mid; hit_ix = ix; break; }
                if (c < 0) lo = mid + 1; else hi = mid;
            }
        }
        if (bad) { rejects |= kLookupCorrupt; break; } // the reference's read_at would fail here: the whole get errors out
    }
    if constexpr (kEmit) {
        uint32_t d = kScanNone;
        uint4 rec = make_uint4(0, 0, 0, 0);
        if (found_table >= 0) {
            const TableDesc &t = p.tables[found_table];
            const uint64_t off = (uint64_t)hit_ix.x | ((uint64_t)hit_ix.y << 32); // off + 8 + klen <= data_len: probe checked it
            const uint64_t ks = hit_ix.z, fs = hit_ix.w;
            bool ok = ks == 8 + klen && fs >= ks + 24 && fs <= t.data_len - off;
            if (ok) {
                const uint8_t *e = t.data + off;
                ok = ld_bytes_le<true>(e + ks, 8) == fs - ks - 24 &&
                     ts_decodes(ld_bytes_le<true>(e + fs - 16, 8), ld_bytes_le<true>(e + fs - 8, 8));
            }
            if (ok) {
                d = 0;
                const unsigned long long src = reinterpret_cast<unsigned long long>(t.data + off);
                rec = make_uint4((uint32_t)src, (uint32_t)(src >> 32), (uint32_t)ks, (uint32_t)fs);
            } else {
                rejects |= kLookupBadEntry;
            }
        }
        em.dest[q] = d;
        em.flat[q] = rec;
    }
    p.out[q] = make_uint4((uint32_t)found_table, rejects, (uint32_t)record, (uint32_t)(record >> 32));
}

__global__ void __launch_bounds__(256, DBEEL_LOOKUP_MINB) k_lookup(LookupParams p) {
    pdl_trigger();
    pdl_wait();
    lookup_query<false>(p, LookupEmit{nullptr, nullptr});
}

__global__ void __launch_bounds__(256, DBEEL_LOOKUP_MINB) k_lookup_emit(LookupParams p, LookupEmit em) {
    pdl_trigger();
    pdl_wait();
    lookup_query<true>(p, em);
}

} // namespace dbeel
