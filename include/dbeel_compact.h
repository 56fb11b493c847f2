/*
 * dbeel_compact.h -- C ABI of the H100 compaction engine (libdbeel_compact.so).
 *
 * This is the drop-in boundary for ONE hot path of tontinton/dbeel's storage engine: the
 * merge core of LSMTree::compact, the memtable flush that feeds level 0, and the
 * bloom / per-entry index build on the output run.  Everything else (file open/create,
 * the CompactionAction journal, renames, the sstables swap, the page cache, the WAL)
 * stays with the caller.  The library never touches the filesystem.
 *
 * Reference interfaces replaced (paths under /root/reference):
 *
 *   dbeel_compact*      <- the body of LSMTree::compact between opening the inputs and
 *                          writing the bloom file: src/storage_engine/lsm_tree.rs:1002-1076
 *                          (BinaryHeap<CompactionItem> merge :52-71,:1038-1066,
 *                          read_next_entry :1158-1170, EntryWriter::write/close
 *                          src/storage_engine/entry_writer.rs:71-160, Bloom::set + dump
 *                          lsm_tree.rs:1026-1034,:1049-1051,:1070-1076)
 *   dbeel_flush*        <- RedBlackTree::set semantics (rbtree_arena/src/lib.rs:497-534) +
 *                          LSMTree::flush_memtable_to_disk (lsm_tree.rs:925-946)
 *   dbeel_flush_many*   <- the same for many memtables at once (several collections / shards, or a backlog)
 *   dbeel_compact_many* <- compact_tree's loop over the groups its picker produced: one LSMTree::compact per
 *                          group (src/tasks/compaction.rs:82-101), all groups in one launch sequence
 *   dbeel_compact_stream<- the same merge core with the reference's file edge around it: the DmaStreamReaders of the
 *                          inputs (lsm_tree.rs:984-991) and EntryWriter's DMA files (entry_writer.rs:30-69) become
 *                          read / write callbacks feeding a pinned ring                 ["next" row N3]
 *   dbeel_get_many*     <- the SSTable loop of LSMTree::get_entry: Bloom::check + binary_search
 *                          (lsm_tree.rs:605-670, 686-719) for a batch of keys        ["next" row N2]
 *   dbeel_get_values*   <- the same, returning the entries binary_search decodes (:628-651)
 *   dbeel_wal_flush*    <- read_memtable_from_wal_file + the recovery flush of open_or_create_ex
 *                          (lsm_tree.rs:552-574, 478-513)                            ["next" row N4]
 *   dbeel_scan*         <- the SSTable part of LSMTree::iter_filter (lsm_tree.rs:133-282) with migrate_actions' hash-range
 *                          filter (src/tasks/migration.rs:54-131) or a key range                ["next" row N5]
 *   dbeel_bloom_*       <- Bloom::new_for_fp_rate sizing (lsm_tree.rs:1028-1031)
 *   error codes         <- src/error.rs:8-74 (only the variants this path can raise)
 *
 * Byte formats are the reference's own (bincode fixint little-endian, mod.rs:45-73):
 *   .data  record = klen:u64 | key | dlen:u64 | data | ts:i128      (dlen == 0: tombstone)
 *   .index record = offset:u64 | key_size:u32 (=8+klen) | full_size:u32   (16 bytes)
 *   .bloom        = bincode(bloomfilter::Bloom) -- see DESIGN.md for the field order
 *
 * Plain pointers and sizes only; no C++ or torch types cross this boundary.
 */
#ifndef DBEEL_COMPACT_H
#define DBEEL_COMPACT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DBEEL_ABI_VERSION 1

/* status codes (0 = ok).  No exception or panic ever crosses the ABI. */
enum {
    DBEEL_OK = 0,
    DBEEL_ERR_INVALID_ARG = 1,     /* null pointer, misaligned device buffer, bad option    */
    DBEEL_ERR_CAPACITY = 2,        /* an output buffer is smaller than dbeel_compact_bound  */
    DBEEL_ERR_ITEM_TOO_LARGE = 3,  /* Error::ItemTooLarge, entry_writer.rs:72-74            */
    DBEEL_ERR_CUDA = 4,            /* a CUDA call failed; dbeel_last_error() has the text   */
    DBEEL_ERR_NOMEM = 5,           /* device or pinned-host allocation failed               */
    DBEEL_ERR_TOO_MANY_RUNS = 6,   /* more than DBEEL_MAX_RUNS inputs                       */
    DBEEL_ERR_TOO_MANY_ENTRIES = 7,/* more than 2^32-2 input entries in one job             */
    DBEEL_ERR_UNSORTED_RUN = 8,    /* an input run violates "keys strictly ascending"       */
    DBEEL_ERR_NO_DEVICE = 9,       /* no CUDA device / not an sm_90 part                    */
    DBEEL_ERR_BUSY = 10,           /* another call holds the engine, or a submitted job is  */
                                   /* unreaped (then err / stats stay the job's)            */
    DBEEL_ERR_BAD_BLOOM = 11,      /* a .bloom file is not a bincode bloomfilter::Bloom      */
    DBEEL_ERR_TREE_FULL = 12       /* rbtree_arena ReachedCapacity (lib.rs:458-461)          */
};

#define DBEEL_MAX_RUNS 1024u
#define DBEEL_INDEX_ENTRY_SIZE 16u            /* mod.rs:33 */
#define DBEEL_DEFAULT_BLOOM_MIN_SIZE 1048576u /* mod.rs:19 */
#define DBEEL_DEFAULT_BLOOM_FP 0.01           /* lsm_tree.rs:48 */
#define DBEEL_DEFAULT_TREE_CAPACITY 8192u     /* mod.rs:18 */

/* One input SSTable: the bytes of its .data and .index files.
 * For the *_device entry points both are device pointers; `index` must be aligned to 16 bytes, `data` may start anywhere
 * (the SSTables dbeel_flush_many / dbeel_compact_many leave back to back in one output stream are valid inputs as they lie). */
typedef struct dbeel_run {
    const void *data;
    uint64_t data_len;
    const void *index;
    uint64_t index_len; /* entries = index_len / 16 (lsm_tree.rs:978-979); a ragged tail is ignored */
} dbeel_run;

/* Output SSTable buffers, owned by the caller.  *_cap in, *_len out. */
typedef struct dbeel_out {
    void *data;
    uint64_t data_cap, data_len;
    void *index;
    uint64_t index_cap, index_len;
    void *bloom;         /* may be NULL when bloom_cap == 0 (no bloom will be produced) */
    uint64_t bloom_cap, bloom_len; /* bloom_len == 0: no .bloom file (lsm_tree.rs:1026-1034) */
    uint64_t items_written;        /* lsm_tree.rs:1053 */
} dbeel_out;

#define DBEEL_FLAG_VERIFY_SORTED 0x1u /* full adjacent-key check of every input run */
/* Decode the input runs exactly like the reference's sequential reader (read_next_entry, lsm_tree.rs:1158-1170):
 *   - an index record's `offset` and `key_size` are IGNORED -- the entry is the next full_size bytes of the .data stream
 *     and its key length is the bincode length prefix found there (the output .index carries the recomputed values,
 *     entry_writer.rs:76-86);
 *   - an i128 timestamp outside `time`'s +-9999-year range fails the decode (utils/timestamp_nanos.rs:15-24) and, like
 *     every decode error, ends that run (lsm_tree.rs:1014,1063).
 * Without the flag the engine is stricter about the index (a wrong offset / key_size ends the run) and does not range-
 * check timestamps; on files the reference's own writer produced both modes give byte-identical output.
 * dbeel_compact / dbeel_compact_device / dbeel_compact_submit only. */
#define DBEEL_FLAG_REFERENCE_READER 0x2u

typedef struct dbeel_compact_opts {
    int32_t keep_tombstones;   /* LSMTree::compact's third argument (lsm_tree.rs:954)      */
    uint32_t flags;            /* DBEEL_FLAG_*                                             */
    uint64_t bloom_min_size;   /* --sstable-bloom-min-size, strict '>' (lsm_tree.rs:1027)  */
    double bloom_fp;           /* BLOOM_MAX_ALLOWED_ERROR                                  */
    const uint8_t *bloom_seed; /* 32 bytes (host memory), or NULL = random like getrandom  */
} dbeel_compact_opts;

/* What the last job did.  Times are CUDA-event milliseconds on the engine's stream. */
typedef struct dbeel_stats {
    uint64_t input_bytes;      /* sum(len(.data)+len(.index))                              */
    uint64_t output_bytes;     /* len(out.data)+len(out.index)+len(out.bloom)              */
    uint64_t entries_in;       /* sum(index_len/16)                                        */
    uint64_t entries_valid;    /* after run truncation at the first undecodable record     */
    uint64_t entries_out;      /* items_written                                            */
    uint32_t runs_truncated;   /* runs that ended early (lsm_tree.rs:1014,1063)            */
    uint32_t key_prefix_len;   /* common key prefix skipped by the comparison window        */
    uint32_t merge_passes;
    uint32_t kernel_launches;  /* kernels launched by this job                             */
    float ms_total;            /* first kernel .. last kernel (device-resident part)       */
    float ms_extract;          /* validate + key-window extraction                         */
    float ms_merge;            /* all merge passes                                         */
    float ms_resolve;          /* winner / tombstone resolution + offsets scan + .index    */
    float ms_gather;           /* .data gather + bloom (the roofline kernel)               */
    float ms_h2d, ms_d2h;      /* host entry points only                                   */
    uint64_t gather_bytes;     /* algorithmic bytes of the gather kernel (read + written)  */
    uint32_t partitions;       /* host entry points: key-range partitions pipelined (1 = single shot) */
    uint32_t index_repaired;   /* DBEEL_FLAG_REFERENCE_READER: 1 = an input index disagreed with its .data and the job ran on the canonical index */
} dbeel_stats;

typedef struct dbeel_engine dbeel_engine;

/* One engine per calling thread / shard, bound to one GPU and one stream. */
int dbeel_engine_create(int device, dbeel_engine **out);
void dbeel_engine_destroy(dbeel_engine *e);
/* The engine's CUDA stream (a cudaStream_t): every kernel of its jobs is launched there.  For callers that want to record
 * their own events around jobs or order other work against them.  Several engines on one GPU run their jobs concurrently. */
void *dbeel_engine_stream(dbeel_engine *e);

/* Host placement.  dbeel pins one executor thread per core (src/main.rs:51-60); with one GPU per shard that thread and
 * the pinned buffers it stages through should sit on the GPU's NUMA node, or every byte crosses the socket interconnect on
 * its way to the PCIe root complex.  dbeel_bind_to_gpu moves the CALLING thread onto the CPUs of `device`'s NUMA node
 * (within the process's allowed set) and prefers that node for its future page allocations; call it before
 * dbeel_host_alloc / before touching the buffers.  numa_node / n_cpus (nullable) report what was applied (-1 / 0 when the
 * machine exposes no NUMA topology: not an error). */
int dbeel_gpu_numa_node(int device);
int dbeel_bind_to_gpu(int device, int *numa_node, int *n_cpus);

/* Upper bounds for the output buffers of a compaction of `runs` (host-side arithmetic only):
 * data_cap = sum(data_len), index_cap = 16 * sum(index_len/16), bloom_cap = size of the
 * .bloom file or 0 when sum(data_len) <= bloom_min_size. */
int dbeel_compact_bound(const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts,
                        uint64_t *data_cap, uint64_t *index_cap, uint64_t *bloom_cap);

/* Merge `runs` (runs[i] is position i in indices_to_compact: the final tie-break) into one
 * SSTable.  Host buffers in, host buffers out; copies are part of the call. */
int dbeel_compact(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs,
                  const dbeel_compact_opts *opts, dbeel_out *out);

/* The same compaction fed from files ["next" row N3: the storage edge].  The reference reads its inputs through
 * DmaStreamReaders (lsm_tree.rs:984-991) and writes through EntryWriter's buffered DMA files (entry_writer.rs:30-69); here
 * the caller hands over two callbacks instead of buffers, and the engine moves the bytes
 *     file -> read() -> pinned ring -> H2D -> kernels -> D2H -> pinned ring -> write() -> file
 * one key-range partition at a time, so file reads, both PCIe directions and file writes overlap and the page-locked
 * memory is a few partitions however large the SSTables are.  runs[i].data / .index are ignored (lengths only).
 *   read : fill dst with [offset, offset + len) of run `run`'s .data (DBEEL_STREAM_DATA) or .index (DBEEL_STREAM_INDEX)
 *   write: store len bytes at `offset` of the output's .data / .index / .bloom (DBEEL_STREAM_BLOOM: one call, offset 0)
 * Both are called from several engine threads at once (pread / pwrite are fine) and return 0 or an error code of the
 * caller's, which dbeel_compact_stream returns unchanged.  Output pieces arrive in no particular order; when an input turns
 * out to need the one-piece path (a run that ends early, lsm_tree.rs:1014,1063) the outputs are written again from offset
 * 0, so the caller truncates each output to out->*_len afterwards (bloom_len == 0: no .bloom file).  `out` returns
 * lengths only; its pointers are ignored.  Same bytes as dbeel_compact. */
#define DBEEL_STREAM_DATA 1u  /* = FileTypeKind::Data  (mod.rs:36-42) */
#define DBEEL_STREAM_INDEX 2u /* = FileTypeKind::Index */
#define DBEEL_STREAM_BLOOM 3u /* = FileTypeKind::Bloom */
typedef struct dbeel_stream_io {
    int (*read)(void *ctx, uint32_t run, uint32_t kind, uint64_t offset, uint64_t len, void *dst);
    int (*write)(void *ctx, uint32_t kind, uint64_t offset, const void *src, uint64_t len);
    void *ctx;
} dbeel_stream_io;
int dbeel_compact_stream(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts,
                         const dbeel_stream_io *io, dbeel_out *out);

/* Same, inputs and outputs resident in device memory (16-byte aligned).  Returns after the
 * job has completed on the engine's stream. */
int dbeel_compact_device(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs,
                         const dbeel_compact_opts *opts, dbeel_out *out);

/* Memtable flush: `batch` holds writes in ARRIVAL order in run layout (keys may repeat, not
 * sorted).  Output = what flush_memtable_to_disk writes for the memtable those writes
 * build: ascending keys, last arrival per key, tombstones kept, no bloom.  The caller cuts
 * batches at memtable boundaries (dbeel_memtable_cut helps). */
int dbeel_flush(dbeel_engine *e, const dbeel_run *batch, dbeel_out *out);
int dbeel_flush_device(dbeel_engine *e, const dbeel_run *batch, dbeel_out *out);

/* Many memtables in one launch sequence (the flush side of a write-heavy shard produces a memtable every few
 * milliseconds; one job per memtable is launch-bound).  batches[i] is memtable i's arrivals (same layout as
 * dbeel_flush).  The n SSTables are written back to back into out->data / out->index; table[i] says where
 * SSTable i lives.  Every SSTable's .index offsets are relative to its own .data start, exactly what n separate
 * dbeel_flush calls would have produced. */
typedef struct dbeel_flush_table {
    uint64_t data_off, data_len;   /* bytes of out->data holding this memtable's .data file   */
    uint64_t index_off, index_len; /* bytes of out->index holding its .index file             */
    uint64_t items;                /* entries written (distinct keys of the memtable)          */
} dbeel_flush_table;
int dbeel_flush_many(dbeel_engine *e, const dbeel_run *batches, uint32_t n_batches, dbeel_out *out,
                     dbeel_flush_table *table /* n_batches rows, host memory */);
int dbeel_flush_many_device(dbeel_engine *e, const dbeel_run *batches, uint32_t n_batches, dbeel_out *out,
                            dbeel_flush_table *table);

/* ---- cfg5: shard routing + flushes of routed streams ---------------------------------------------------------------
 * A dbeel node runs one shard per core; a key belongs to the shard that owns murmur3_32(key bytes, seed 0) on the
 * consistent-hash ring of shard names "<node name>-<cpu id>" (hash_bytes / hash_string, src/shards.rs:95-101; names
 * :213-214).  MyShard::owns_key with replica_index 0 (shards.rs:586-598, checked per request in
 * src/tasks/db_server.rs:119-122): shard s owns the hashes in [hash of the previous shard on the ring, hash of s), wrapping
 * -- i.e. the first shard whose hash is GREATER than the key's.  (dbeel_client picks the first shard with hash >= the key's,
 * dbeel_client/src/lib.rs:344; the two differ only for a key whose hash equals a shard's, which that shard refuses.) */
#define DBEEL_MAX_SHARDS 256u
uint32_t dbeel_murmur3_32(const void *bytes, uint64_t len, uint32_t seed);                 /* host arithmetic */
uint32_t dbeel_ring_owner(const uint32_t *ring_hashes, uint32_t n_shards, uint32_t key_hash); /* host arithmetic: ring position */
/* Build the ring of `n_shards` shards of node `node_name` (NULL = "dbeel", args.rs): ring_hashes[] ascending,
 * ring_ids[p] = cpu id of the shard at ring position p.  Returns 0, or DBEEL_ERR_INVALID_ARG on a hash collision. */
int dbeel_shard_ring(const char *node_name, uint32_t n_shards, uint32_t *ring_hashes, uint32_t *ring_ids);

/* Route an arrival batch (run layout, arrival order; device pointers, 16-byte aligned) to the ring's shards on the GPU.
 * out_index (device, >= batch->index_len bytes) receives the batch's index records split into one stream per ring
 * position: position p's arrivals, in arrival order, are records [sum(counts[0..p)), +counts[p]).  The records are
 * unchanged -- they still point into batch->data -- so a shard's stream is an arrival batch with sparse offsets (below).
 * shard_of (device, n u32, or NULL) receives every arrival's ring position; counts / payload_bytes (host, n_shards each;
 * payload_bytes may be NULL) the arrivals and the sum of full_size per position.
 * out_key_hash64 (device, n u64, or NULL): a 64-bit identity of every arrival's key, in the same shard-major order as
 * out_index -- the input of dbeel_memtable_cuts_device. */
int dbeel_route_device(dbeel_engine *e, const dbeel_run *batch, const uint32_t *ring_hashes /* host, ascending */,
                       uint32_t n_shards, void *out_index, uint64_t out_index_cap, uint32_t *shard_of, void *out_key_hash64,
                       uint64_t *counts, uint64_t *payload_bytes);

/* The memtable-full trigger (lsm_tree.rs:747-765, 600-603: a flush starts right after the insert that makes the tree hold
 * `capacity` keys) for whole streams at once, on the device.  Stream s = key identities [stream_starts[s],
 * stream_starts[s+1]) of key_hash64 (arrival order).  cuts[cut_starts[s] .. cut_starts[s+1]) receive, for every FULL memtable
 * of stream s, the number of the stream's arrivals consumed up to and including it; what follows the last cut is the
 * memtable still filling.  capacity <= 9216 (shared-memory set); max_cuts_total >= sum(len(s) / capacity).
 * The identities are 64-bit hashes: a collision inside one memtable would cut one key late.  The flush reports every
 * SSTable's exact entry count -- a full memtable must yield exactly `capacity` -- so callers check that and fall back to the
 * exact host function dbeel_memtable_cut (dbeel_tree.h) on a mismatch. */
int dbeel_memtable_cuts_device(dbeel_engine *e, const void *key_hash64, const uint64_t *stream_starts /* host */,
                               uint32_t n_streams, uint32_t capacity, uint32_t *cuts /* host */, uint32_t *cut_starts /* host */,
                               uint32_t max_cuts_total);

/* dbeel_flush_many_device for batches whose index records do not abut in .data (slices of a routed stream: every batch's
 * `data` is the shared arrival buffer, `index` a slice of dbeel_route_device's out_index).  payload_bound >= the sum of
 * full_size over all batches (e.g. from payload_bytes above); out->data_cap >= payload_bound.  DBEEL_ERR_CAPACITY if the
 * bound turns out too low (nothing is written past it). */
int dbeel_flush_many_sparse_device(dbeel_engine *e, const dbeel_run *batches, uint32_t n_batches, uint64_t payload_bound,
                                   dbeel_out *out, dbeel_flush_table *table);

/* ---- N1: many independent compactions in one launch sequence ---------------------------------------------------
 * compact_tree (src/tasks/compaction.rs:82-101) issues one LSMTree::compact per group of SSTables it picked, and a node
 * runs one such loop per collection and shard; small level-0 merges are launch-bound one at a time.  Every job here is
 * exactly one dbeel_compact: its own runs (tie-break = position inside the job), its own keep_tombstones, its own bloom
 * filter (enabled and sized from ITS inputs, its own 32-byte seed).  Outputs land back to back in out->data /
 * out->index (file-relative .index offsets per job) and in out->bloom at 16-byte aligned offsets; results[j] says where.
 * Each job's three files are byte-identical to a separate dbeel_compact with the same arguments. */
typedef struct dbeel_job {
    const dbeel_run *runs;     /* in the order of indices_to_compact */
    uint32_t n_runs;
    int32_t keep_tombstones;
    const uint8_t *bloom_seed; /* 32 bytes, or NULL = fresh random seed */
} dbeel_job;
typedef struct dbeel_job_result {
    uint64_t data_off, data_len;
    uint64_t index_off, index_len;
    uint64_t bloom_off, bloom_len; /* bloom_len == 0: no filter for this job (lsm_tree.rs:1026-1034) */
    uint64_t items_written;
} dbeel_job_result;
int dbeel_compact_many_bound(const dbeel_job *jobs, uint32_t n_jobs, uint64_t bloom_min_size, double bloom_fp,
                             uint64_t *data_cap, uint64_t *index_cap, uint64_t *bloom_cap);
int dbeel_compact_many(dbeel_engine *e, const dbeel_job *jobs, uint32_t n_jobs, uint64_t bloom_min_size, double bloom_fp,
                       dbeel_out *out, dbeel_job_result *results);
int dbeel_compact_many_device(dbeel_engine *e, const dbeel_job *jobs, uint32_t n_jobs, uint64_t bloom_min_size,
                              double bloom_fp, dbeel_out *out, dbeel_job_result *results);

/* Asynchronous form of dbeel_compact for callers that must not block their reactor (dbeel's
 * compaction task runs on a glommio executor, src/tasks/compaction.rs:139-153): submit returns at
 * once, the job runs on an engine-owned worker thread, poll / wait report its status.  All
 * buffers (runs, the 32-byte seed, out) must stay valid until the job has been reaped by a
 * dbeel_wait() or a dbeel_poll() that returned 1.  One job per engine at a time (DBEEL_ERR_BUSY). */
int dbeel_compact_submit(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs,
                         const dbeel_compact_opts *opts, dbeel_out *out);
int dbeel_poll(dbeel_engine *e, int *status); /* returns 1 when finished (then *status = the job's code), else 0 */
int dbeel_wait(dbeel_engine *e);              /* blocks; returns the job's status code */

/* ---- N2: batched point lookups on the files this engine writes ------------------------------------------------
 * Replaces the SSTable loop of LSMTree::get_entry (src/storage_engine/lsm_tree.rs:686-719) for a batch of keys:
 * tables[] is the tree's `sstables` vector (oldest first; the loop walks it newest first, :688), every table is its
 * three files' bytes.  Per key: Bloom::check on the .bloom bytes (:691-696), then binary_search over .index / .data
 * (:605-670).  The memtable look-ups in front of it (:677-684) stay on the host.
 *
 *   DBEEL_LOOKUP_REFERENCE  binary_search restated step for step.  Its loop leaves right after probing index record 0
 *                           (`if half == 0 ... break`, :660), so a few present keys are reported absent -- this mode
 *                           reports exactly what the reference reports.
 *   DBEEL_LOOKUP_EXACT      lower-bound search: every present key is found.                                        */
#define DBEEL_LOOKUP_REFERENCE 0u
#define DBEEL_LOOKUP_EXACT 1u
#define DBEEL_LOOKUP_CORRUPT 0x80000000u /* in bloom_rejects: an index record pointed outside its .data file (the
                                            reference's read_at fails there and the whole get returns Err) */
typedef struct dbeel_table {
    const void *data;  uint64_t data_len;
    const void *index; uint64_t index_len;  /* multiple of 16 */
    const void *bloom; uint64_t bloom_len;  /* the .bloom file, or NULL / 0 when the table has none (:94-101) */
} dbeel_table;
typedef struct dbeel_lookup_result {
    int32_t table;          /* position in tables[] of the SSTable that answered, -1 = key not found      */
    uint32_t bloom_rejects; /* tables skipped by their filter before the answer (| DBEEL_LOOKUP_CORRUPT)    */
    uint64_t record;        /* index record number inside that table: its EntryOffset locates the entry    */
} dbeel_lookup_result;
/* keys: the query keys back to back; key_offsets: n_keys + 1 byte offsets (key i = keys[key_offsets[i] ..
 * key_offsets[i+1])).  dbeel_get_many takes host pointers everywhere and uploads the tables for the call (tests,
 * small tables); dbeel_get_many_device takes device pointers everywhere (tables resident in HBM, e.g. straight
 * from dbeel_compact_device) -- only the 172-byte trailer of each .bloom is read back to parse its parameters. */
int dbeel_get_many(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys,
                   const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode, dbeel_lookup_result *results);
int dbeel_get_many_device(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys,
                          const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode, dbeel_lookup_result *results);

/* Batched reads that return the entries: the rows of dbeel_get_many for the same arguments, plus the entry every
 * answered row names (what get_entry returns, :674-723), so nothing is read a second time.
 * A row answers when table >= 0 and its hit decodes the way binary_search decodes one (:628-651): read_at(offset,
 * key_size) is exactly the key (key_size == 8 + klen), and read_at(offset + key_size, full_size - key_size) exactly one
 * EntryValue (u64 dlen | data | i128 timestamp, 8 + dlen + 16 == full_size - key_size) inside .data, with the timestamp
 * inside `time`'s +-9999 years.  A hit that does not decode gets DBEEL_LOOKUP_BAD_ENTRY and no entry, and no older table
 * is tried (the reference's get returns Err).  The search itself is dbeel_get_many's (key_size is not read while probing).
 * out->data / out->index receive one entry per answered row, in query order, bytes as stored (a tombstone comes back with
 * dlen == 0 and its timestamp; a key asked twice comes back twice): an arrival batch whose .index offsets start at 0, like
 * a scan destination.  out->items_written = entries; row i's entry is entry number (answered rows before i).
 * Caps: the sum of full_size over the hits is enough.  When out->data_cap or out->index_cap is smaller than needed:
 * DBEEL_ERR_CAPACITY, out->data_len / index_len = the sizes needed, the rows filled, nothing written to out.
 * Limits: n_keys < 2^32 - 16 (DBEEL_ERR_INVALID_ARG).  out->bloom is not used.  dbeel_get_values takes host memory (tables uploaded whole, only the rows and the selected bytes come
 * back); dbeel_get_values_device takes device memory for tables, keys, offsets, results and out (out 16-byte aligned). */
#define DBEEL_LOOKUP_BAD_ENTRY 0x40000000u /* in bloom_rejects: the hit's entry does not decode (get_entry returns Err) */
int dbeel_get_values(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys,
                     const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode, dbeel_out *out,
                     dbeel_lookup_result *results);
int dbeel_get_values_device(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys,
                            const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode, dbeel_out *out,
                            dbeel_lookup_result *results);

/* ---- N5: scans -- LSMTree::iter_filter over a tree's SSTables ------------------------------------------------------
 * Replaces the SSTable part of AsyncIter (src/storage_engine/lsm_tree.rs:133-282, iter_filter :1183-1189) with its filter
 * for the two uses the reference has: migration (migrate_actions, src/tasks/migration.rs:62-131: murmur3_32 of the key in
 * one of a list of hash ranges) and key-range reads ([start, end) in Vec<u8> order, lsm_tree.rs:1363-1397).
 * tables[] is the tree's `sstables` vector, oldest first, read in that order; every table's floor(index_len / 16) records in
 * order, each entry read at its EntryOffset's (offset, full_size) -- key_size is ignored, offsets need not be running.  No
 * dedupe, no tombstone rule: duplicates across tables and tombstones come out as stored.  The memtable part of the
 * iterator (emitted after the tables, :155-173) stays with the caller.
 *
 * Every accepted entry goes to the FIRST range that accepts it:
 *   DBEEL_SCAN_HASH  ranges = uint32_t[2 * n_ranges] (start, end) pairs; range d accepts murmur3_32(key, 0) = h when
 *                    between_cmp(h, start, end) (migration.rs:54-60, restated literally: for end < start every hash, for
 *                    start == end none).
 *   DBEEL_SCAN_KEY   ranges = a dbeel_key_ranges: range d accepts start_d <= key < end_d.
 * Destination d's entries are written, in iteration order, as one SSTable pair: results[d] says where it lies in out->data /
 * out->index (file-relative .index offsets, key_size = 8 + key length, bloom_len = 0).  Each pair is a valid arrival
 * batch for dbeel_flush / dbeel_route_device.
 *
 * The reference decodes before it filters (lsm_tree.rs:273), so the first record that does not decode ends the scan even
 * where no range would have taken it; what precedes it is delivered.  *stop reports it:
 *   DBEEL_SCAN_STOP_ERR    next() returns Err: the entry is not exactly one bincode Entry of full_size bytes, or its
 *                          timestamp is outside time's +-9999 years (utils/timestamp_nanos.rs:15-24).
 *   DBEEL_SCAN_STOP_PANIC  the reference panics: full_size == 0 (cached_file_reader.rs:82), bytes past the end of .data
 *                          (:68), or a table with no index record (its first index read runs past EOF).
 * Limits: n_tables <= DBEEL_MAX_RUNS, 1 <= n_ranges <= DBEEL_MAX_SCAN_RANGES, fewer than 2^32 - 16 records in all; else
 * DBEEL_ERR_INVALID_ARG.  Output caps: dbeel_scan_bound (entries whose index records overlap can exceed it:
 * DBEEL_ERR_CAPACITY, nothing written).  The tables' bloom fields are ignored.
 * dbeel_scan takes host memory and uploads the tables whole; dbeel_scan_device takes device pointers for tables / out
 * (.index 16-byte aligned, outputs 16-byte aligned), ranges / results / stop stay in host memory in both. */
#define DBEEL_SCAN_HASH 0u
#define DBEEL_SCAN_KEY 1u
#define DBEEL_MAX_SCAN_RANGES 256u
#define DBEEL_SCAN_STOP_NONE 0u
#define DBEEL_SCAN_STOP_ERR 1u
#define DBEEL_SCAN_STOP_PANIC 2u
typedef struct dbeel_key_ranges {
    const void *keys;            /* start_d = keys[off[2d] .. off[2d+1]), end_d = keys[off[2d+1] .. off[2d+2]) */
    const uint64_t *key_offsets; /* 2 * n_ranges + 1 byte offsets */
} dbeel_key_ranges;
typedef struct dbeel_scan_stop {
    int32_t table;   /* position in tables[] of the first failing record, -1 = the scan read every record */
    uint32_t reason; /* DBEEL_SCAN_STOP_* */
    uint64_t record; /* its index record number in that table */
} dbeel_scan_stop;
/* data_cap = sum(data_len), index_cap = sum(index_len) (host arithmetic only) */
int dbeel_scan_bound(const dbeel_table *tables, uint32_t n_tables, uint64_t *data_cap, uint64_t *index_cap);
int dbeel_scan(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges,
               uint32_t n_ranges, dbeel_out *out, dbeel_job_result *results, dbeel_scan_stop *stop);
int dbeel_scan_device(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges,
                      uint32_t n_ranges, dbeel_out *out, dbeel_job_result *results, dbeel_scan_stop *stop);

/* The same scan fed from files, for trees of any size (LSMTree::iter_filter's SSTable part, lsm_tree.rs:210-281): migration
 * reads a shard's whole tree, which is the tree that grows until the node is rebalanced.  The engine moves the bytes
 *     file -> read() -> pinned ring -> H2D -> kernels -> D2H -> pinned ring -> write() -> file
 * one partition at a time: a partition is a contiguous run of records in iteration order (it may span tables) with, per
 * table, its index slice and the .data window that holds them.  Device and page-locked memory are bounded by the partition
 * budget (DBEEL_PARTITION_MB / DBEEL_PARTITION_KB) and the ring depth (DBEEL_STREAM_RING), not by the tree; the planner reads
 * the .index files in pieces and keeps one row per partition.  tables[i].data / .index are ignored (lengths only).
 *   read : as dbeel_stream_io.read: [offset, offset + len) of table `table`'s .data (DBEEL_STREAM_DATA) or .index
 *          (DBEEL_STREAM_INDEX).  The .index files are read twice: once to plan, once into the ring.
 *   write: len bytes at `offset` of destination `dest`'s .data (DBEEL_STREAM_DATA) or .index (DBEEL_STREAM_INDEX) file.
 *          Every destination's two files start at offset 0 (.index offsets are relative to its own .data file); pieces
 *          arrive in any order, from several threads, at their final offsets.
 * Both return 0 or an error code of the caller's, which dbeel_scan_stream returns unchanged; the engine stays usable.
 * results[d]: data_len / index_len / items_written of destination d's files, *_off = 0, bloom_len = 0.  The files and
 * *stop are byte-identical to what dbeel_scan returns for the same tables (stop in (table, record) of tables[]).  Only the
 * selected bytes cross PCIe back; dbeel_last_stats reports input_bytes = bytes copied to the device (windows, index slices,
 * table headers), output_bytes = the selected output, partitions = partitions run.
 * Limits and argument checks as dbeel_scan, except that the record limit (fewer than 2^32 - 16) applies per partition, not
 * to the tree. */
typedef struct dbeel_scan_io {
    int (*read)(void *ctx, uint32_t table, uint32_t kind, uint64_t offset, uint64_t len, void *dst);
    int (*write)(void *ctx, uint32_t dest, uint32_t kind, uint64_t offset, const void *src, uint64_t len);
    void *ctx;
} dbeel_scan_io;
int dbeel_scan_stream(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges,
                      uint32_t n_ranges, const dbeel_scan_io *io, dbeel_job_result *results, dbeel_scan_stop *stop);

/* dbeel_get_values on tables that stay in files: the same rows (DBEEL_LOOKUP_CORRUPT and DBEEL_LOOKUP_BAD_ENTRY included),
 * the same out->data / out->index / items_written, the same DBEEL_ERR_CAPACITY behaviour, argument checks and limits, in
 * both modes and on damaged tables -- but only the parts of .data and .index the batch's searches reach are read, which is
 * what the reference reads per get: about log2(n) index records and key frames per table its filter lets through, plus
 * the entry that answers (binary_search, lsm_tree.rs:605-670).
 * tables[i].data_len / index_len give the file sizes (.data / .index pointers are ignored); tables[i].bloom is the .bloom
 * file in host memory or NULL, as the reference keeps it in memory.  .data and .index are read only through io->read
 * (io->write is not used and may be NULL), from the engine's reader threads; a nonzero return comes back unchanged and the
 * engine stays usable.  Per table, newest first: the filter runs on the device, a table no open query passes is not read at
 * all; the index records and key frames of the top levels of the search's probe tree are read (ranges that lie close
 * together as one read), the searches descend on them on the device, and the index slices and .data windows of the leaves
 * they end in are read in groups of about the partition budget (DBEEL_PARTITION_MB / _KB).  A hit's entry is copied out of
 * its leaf's window on the device; a hit at a fence gets a one-record read after the last table.  Device and page-locked
 * memory: a group, the fences, O(n_keys) and the answered entries -- not the tables.  A group holds at least one leaf, so
 * one leaf's window can exceed the budget: about data_len / 2^16 bytes on very large tables, or more when a leaf holds
 * multi-megabyte entries.
 * dbeel_last_stats: input_bytes = bytes read through the callback, output_bytes / entries_out as dbeel_get_values,
 * entries_in = n_keys, partitions = leaf groups run.  keys / key_offsets / results / out in host memory. */
int dbeel_get_values_stream(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys,
                            const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode, const dbeel_scan_io *io,
                            dbeel_out *out, dbeel_lookup_result *results);

/* Readers: dbeel_get_values_stream for a serving loop that sends many batches to the same tables.  The reference reads
 * each table's .bloom once, when the table is opened or written (SSTable::new_with_bloom_read, lsm_tree.rs:94-101), and
 * get_entry walks a snapshot of `sstables` (:686-688); a reader does the same for the GPU path:
 *   - dbeel_reader_open validates every .bloom and uploads it once (a bad filter fails the open with the code
 *     dbeel_get_values_stream returns for it); the caller may free its host copies afterwards.  tables / io mean what they
 *     mean for dbeel_get_values_stream, with the same argument checks; io must stay valid until the reader is closed.
 *   - The fences of each table (index record + key frame of the top D_t levels of the probe tree, per mode) are read the
 *     first time a batch in that mode reaches the table, then kept on the device and never read again.  D_t is chosen
 *     per table so that all the reader's fences, both modes, fit fence_bytes (0 = DBEEL_READER_FENCE_BYTES_DEFAULT): the
 *     budget goes one level at a time to the table with the largest leaves, never deeper than 16 levels or log2 of the
 *     table's records.  A cached key frame holds at most DBEEL_READER_FRAME_CAP key bytes.
 *   - A batch descends a table's cached fences when its longest key is at most DBEEL_READER_FRAME_CAP bytes and the depth
 *     dbeel_get_values_stream would read for it is at most D_t.  Otherwise it reads that table's fences for this batch
 *     exactly as dbeel_get_values_stream does.
 * dbeel_reader_get_values returns exactly what dbeel_get_values_stream(e, tables, ..., io, ...) returns for the same keys
 * and mode: the rows (DBEEL_LOOKUP_CORRUPT and DBEEL_LOOKUP_BAD_ENTRY included, damaged tables included), out->data /
 * out->index / items_written, DBEEL_ERR_CAPACITY with the sizes needed, and callback codes unchanged; the reader stays
 * usable after any of them.  dbeel_last_stats: input_bytes = bytes read through the callback in this call (fences loaded
 * on the way included), partitions = leaf groups run, the rest as dbeel_get_values_stream.
 * The reader's device memory (the filters, plus the fences, at most fence_bytes) belongs to the engine.  Open and get
 * take the engine as every entry point does (DBEEL_ERR_BUSY while another call runs).  dbeel_engine_destroy closes the
 * readers still open. */
#define DBEEL_READER_FRAME_CAP 64u
#define DBEEL_READER_FENCE_BYTES_DEFAULT (64ull << 20)
typedef struct dbeel_reader dbeel_reader;
int dbeel_reader_open(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const dbeel_scan_io *io,
                      uint64_t fence_bytes, dbeel_reader **out);
int dbeel_reader_get_values(dbeel_reader *r, const void *keys, const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode,
                            dbeel_out *out, dbeel_lookup_result *results);

/* Batched reads across readers: the point-read batches of many readers (a node's shards and collections, each a tree) in
 * one call.  Batch b asks batches[b].reader for n_keys keys (keys / key_offsets as for dbeel_reader_get_values) in its own
 * mode (DBEEL_LOOKUP_REFERENCE or DBEEL_LOOKUP_EXACT); reserved must be 0.  A reader may appear in several batches, and a
 * batch may have no keys.
 * Result: exactly dbeel_reader_get_values(batches[b].reader, ...) for b = 0, 1, ... in order, concatenated.  results has
 * sum(n_keys) rows in batch order; a row's table is a position in its own reader's tables; the flags and bloom_rejects are
 * the solo call's, on damaged tables too, and one batch's damage or misses never change another batch's rows.  out packs
 * the answered entries in row order as dbeel_get_values packs them: batch b's .data / .index are its solo call's output,
 * appended, its .index offsets shifted by the .data bytes before it; items_written is the total.
 * Reads: the batches run together one table level at a time (level j: every batch's table T_b - 1 - j, newest first), so a
 * level costs one filter, fence and touched-leaf pass for all batches, not one per batch.  Each (batch, table) pair makes
 * its solo call's decisions: cached or per-call fences and their depth, from that batch's longest key and open queries.
 * Every read goes through the pair's own reader's io->read and page cache, and lies inside what the solo calls, made in
 * batch order on readers in the same state, read for that table and file kind: a pair's leaves are loaded in the groups
 * its solo call cuts, and groups of different pairs share a load while they fit the partition budget and each page
 * cache's capacity.  With no page cache, input_bytes is at most the sum of the solo calls'.  A cache whose leaves of one
 * group do not fit it reads them uncached, as a solo call does.
 * Errors leave every reader, the engine and every page cache usable: DBEEL_ERR_INVALID_ARG for null batches / out /
 * results or a null reader, a reader of another engine, n_batches of 0 or above DBEEL_MAX_READER_BATCHES, an unknown mode
 * or nonzero reserved, a null key_offsets, null keys with key bytes, or sum(n_keys) >= 2^32 - 16; DBEEL_ERR_CAPACITY as
 * dbeel_get_values (every row filled, out->data_len / index_len = the sizes needed for the whole call, nothing written);
 * a callback's nonzero return unchanged; DBEEL_ERR_BUSY while another call runs on the engine.
 * dbeel_last_stats: input_bytes = every byte read through every reader's callback, entries_in = sum(n_keys),
 * entries_out / output_bytes = what was returned, partitions = leaf groups run, kernel_launches summed over the call. */
#define DBEEL_MAX_READER_BATCHES 1024u
typedef struct dbeel_reader_batch {
    dbeel_reader *reader;
    const void *keys;            /* as dbeel_reader_get_values */
    const uint64_t *key_offsets; /* n_keys + 1 byte offsets */
    uint64_t n_keys;
    uint32_t mode;               /* DBEEL_LOOKUP_REFERENCE or DBEEL_LOOKUP_EXACT, per batch */
    uint32_t reserved;           /* 0 */
} dbeel_reader_batch;
int dbeel_readers_get_values(dbeel_engine *e, const dbeel_reader_batch *batches, uint32_t n_batches, dbeel_out *out,
                             dbeel_lookup_result *results);

/* Range scans on a reader: dbeel_scan_stream's call on the reader's tables (a snapshot: a tree reader keeps its tables'
 * files open while the tree flushes and compacts).  kind / ranges / n_ranges / results / stop mean what they mean for
 * dbeel_scan_stream, with its argument checks and limits (kind, 1 <= n_ranges <= DBEEL_MAX_SCAN_RANGES, a non-null write,
 * the record limit per partition); ranges, results and stop in host memory.  Output pieces go to write(ctx, ...) as to
 * dbeel_scan_io.write: destination d's .data / .index start at offset 0, pieces arrive in any order and from several
 * threads.  The reader's io.read reads the files; its io.write is not used.  stop->table is a position in the reader's
 * tables.
 *   DBEEL_SCAN_HASH  a hash range cannot seek: exactly what dbeel_scan_stream returns on the reader's tables through the
 *                    reader's io -- the same files, results and stop.
 *   DBEEL_SCAN_KEY   a seek.  For table t of n_t records and each range d with start_d < end_d (byte order), lo = seek_t(start_d)
 *                    and hi = seek_t(end_d); a range with start_d >= end_d takes no record and is not searched.  seek_t(k):
 *                    a = 0, b = n_t; while a < b: mid = a + (b - a) / 2, compare the key of record mid with k (c), a = mid + 1
 *                    if c < 0 else b = mid; the result is a -- the exact-mode search of DBEEL_LOOKUP_EXACT without its exit
 *                    on equality, so the reader's exact-mode fences serve it.  On keys that strictly ascend, seek_t(k) is the
 *                    first record whose key is >= k.  Table t's span is the union of the [lo, hi), merged into ascending
 *                    disjoint record intervals.  The output and *stop are exactly what dbeel_scan_stream (= dbeel_scan)
 *                    returns on the same ranges over the tables cut down to their spans (each .index = its span records back
 *                    to back, .data whole; a table whose span is empty contributes nothing), with record numbers mapped back
 *                    to the original tables.  On the tables the writer produces (keys strictly ascending) with no stop, that
 *                    is plain dbeel_scan_stream(DBEEL_SCAN_KEY) on the same tables, byte for byte.  A table with no index
 *                    record is a DBEEL_SCAN_STOP_PANIC at (t, 0), as in dbeel_scan; nothing is read for it.
 *                    A search that probes a record the lookup reports corrupt (offset or length prefix past the end of .data)
 *                    fails: table t contributes nothing and the scan ends before it, with *stop = (t, reason, r), r the
 *                    smallest such record of t and reason what dbeel_scan reports on reaching r (PANIC when the index record
 *                    alone shows it, ERR otherwise).  Every search finishes before the first record is scanned, so the stop
 *                    is the first, in iteration order, of the failed searches, the empty tables and the stops in the spans.
 *                    Reads: the fences, from the reader's cache under dbeel_reader_get_values' rule (range keys of at most
 *                    DBEEL_READER_FRAME_CAP bytes, the depth for 2 * n_ranges queries at most D_t; a first scan loads the
 *                    exact-mode fences, which get_values shares) or read for this call; the leaves the searches end in (index
 *                    slice and key frames); then the span slices and .data windows, planned and pumped as dbeel_scan_stream
 *                    plans and pumps whole tables.  No other .index or .data byte is read.
 * dbeel_last_stats: input_bytes = bytes read through the callback in this call (fences loaded on the way included; for
 * DBEEL_SCAN_HASH as dbeel_scan_stream), output_bytes as dbeel_scan_stream, entries_in = records in the spans (all records
 * for DBEEL_SCAN_HASH), partitions = span partitions run.  A callback's nonzero return comes back unchanged; the reader
 * stays usable after it, after any stop and after an argument error.  DBEEL_ERR_BUSY while another call runs. */
int dbeel_reader_scan(dbeel_reader *r, uint32_t kind, const void *ranges, uint32_t n_ranges,
                      int (*write)(void *ctx, uint32_t dest, uint32_t kind, uint64_t offset, const void *src, uint64_t len),
                      void *ctx, dbeel_job_result *results, dbeel_scan_stop *stop);

/* Range reads on a reader: what get_entry / dbeel_reader_get_values(DBEEL_LOOKUP_EXACT) return for every key of the
 * ranges, merged on the device.  Let S_d be the entries dbeel_reader_scan(r, DBEEL_SCAN_KEY, ranges, n_ranges, ...)
 * writes to destination d, in its order.
 *   Output.  Destination d receives one SSTable pair: for every distinct key of S_d, in ascending byte order, the LAST
 *            entry of S_d with that key -- on sorted tables the newest table's version, the one get_entry returns.  An
 *            entry with dlen == 0 (a tombstone) is left out unless flags has DBEEL_RANGE_KEEP_TOMBSTONES.  Entries keep
 *            their stored bytes; .index offsets run from 0 and key_size is 8 + klen.  With the flag, destination d is
 *            byte for byte what dbeel_flush writes for S_d taken as one arrival batch.  Every destination is a valid
 *            SSTable (keys strictly ascending), usable as a compaction input or a reader table.
 *   Ranges.  As dbeel_reader_scan(DBEEL_SCAN_KEY): the first range that accepts a key takes it, start >= end takes
 *            nothing, same limits.  DBEEL_ERR_INVALID_ARG for a null write, n_ranges of 0 or more than
 *            DBEEL_MAX_SCAN_RANGES, or an unknown bit in flags.
 *   Stops.   *stop is exactly dbeel_reader_scan's for the same ranges (a failed search, a table with no record, a PANIC or
 *            ERR inside the spans).  With a stop the call returns DBEEL_OK, every results[d] is zero and the bytes already
 *            passed to write are void: a damaged tree's result is its stop, never a merged prefix.
 *   Sorted.  With no stop, a table whose span records (the union of its spans, in record order) do not strictly ascend by
 *            key gives DBEEL_ERR_UNSORTED_RUN, results zero and the bytes written void.  Only tables the writer did not
 *            produce can do that.
 *   Delivery as dbeel_reader_scan: destination d's .data and .index start at offset 0, pieces arrive in any order and
 *            from several threads, the reader's io.write is not used.
 *   Reads.   The bound searches of dbeel_reader_scan (fences cached or read for this call, touched leaves through the page
 *            cache when one is attached); the span .index slices, for planning and again for the partitions; the key-aligned
 *            planner's reads -- a second pass over the span .index slices, the keys of sampled records (.data) and the
 *            searches for those keys, as the bound searches; and the partitions' .data windows (not through the page
 *            cache).  When the span slices and windows fit one partition, the call makes exactly dbeel_reader_scan's reads.
 *   Memory.  Device and page-locked memory are bounded by the partition budget (DBEEL_PARTITION_MB / _KB): a partition's
 *            index slices and windows, and its output bound, are at most the budget plus one record per table, on any
 *            tables.  A partition is a key interval of every table, cut at sampled keys, and a window never spans more
 *            bytes than its records hold.  A key interval that would pass that bound -- possible only when some table's
 *            span keys do not ascend, or when a sampled key's search met a corrupt record -- is not staged: the call
 *            returns dbeel_reader_scan's stop if there is one, else DBEEL_ERR_UNSORTED_RUN.  The searches of the sampled
 *            keys run in batches whose search state fits the budget.
 * dbeel_last_stats: input_bytes = every byte read through the callback in this call, output_bytes / entries_out = what
 * was written (0 with a stop), entries_in = records in the spans, partitions = key partitions run.  A callback's nonzero return comes back
 * unchanged; the reader, the engine and an attached page cache stay usable after every error, stop and argument failure.
 * DBEEL_ERR_BUSY while another call runs. */
#define DBEEL_RANGE_KEEP_TOMBSTONES 0x1u
int dbeel_reader_get_range(dbeel_reader *r, const dbeel_key_ranges *ranges, uint32_t n_ranges, uint32_t flags,
                           int (*write)(void *ctx, uint32_t dest, uint32_t kind, uint64_t offset, const void *src, uint64_t len),
                           void *ctx, dbeel_job_result *results, dbeel_scan_stop *stop);

/* Range reads with a limit, batched: the first entries of many key ranges in one call, for a serving loop (a page of a
 * listing, the next page from a cursor).  Query q is the range [start_q, end_q), laid out as in dbeel_reader_get_range
 * (key_offsets has 2 * n_ranges + 1 entries), with the limit limits[q].  Let G_q be destination 0 of
 * dbeel_reader_get_range(r, &range_q, 1, flags, ...) for that range alone.
 *   Clean.   A query whose range makes that call return no stop and not DBEEL_ERR_UNSORTED_RUN gets the first
 *            min(limits[q], |G_q|) entries of G_q, byte for byte; DBEEL_RANGE_MORE is set iff |G_q| > limits[q].  A query
 *            with start >= end gets count 0, reads nothing and is never stopped, except by an empty table.
 *   Output.  Entries packed as dbeel_get_values packs them: query order, ascending keys within a query, bytes as stored;
 *            the .index offsets start at 0 in out->data, key_size = 8 + klen, out->items_written = the total.  Row q's
 *            entries are entry numbers [first, first + count).  A caller pages on with start = last key + "\x00".
 *   Stops.   A failed bound search or a table with no index record, as seek_t meets them for the query's range alone (the
 *            stop of dbeel_reader_scan's searches): the row is DBEEL_RANGE_STOPPED with that stop and nothing is read for
 *            the query's records.
 *   Damage.  Only a prefix of every span is read.  Let A_q be the merge, under G_q's rule, of every table's span records
 *            for q, each cut just before its first record that fails dbeel_scan's decode (ERR / PANIC as the scan
 *            classifies it) or is not strictly above its predecessor.  The row is then either the first min(limit, |A_q|)
 *            entries of A_q (MORE iff |A_q| > limit), or DBEEL_RANGE_STOPPED with stop = (table, ERR / PANIC, record) of a
 *            record that fails the decode, or DBEEL_RANGE_UNSORTED with stop = (table, DBEEL_SCAN_STOP_NONE, record) of a
 *            record not above its predecessor.  The first record of every non-empty span is always read.  One query's
 *            damage never changes another query's row.
 *   Reads.   The bound searches of the queries with start < end (dbeel_reader_scan's: fences cached or read for this
 *            call, the touched leaves); per query and table, index records from seek_t(start) on, never past
 *            seek_t(end), in chunks that start at seek_t(start) and double for the tables that hold back the merge; the
 *            .data windows of exactly the records staged, each never wider than its records.  Leaf slices, staged index
 *            slices and windows go through an attached page cache.  Nothing else is read.
 *   Memory.  Device and page-locked memory follow the partition budget (DBEEL_PARTITION_MB / _KB): each round runs the
 *            live queries in groups whose staged records (index record, mean entry and workspace) fit it, and a group
 *            holds at least one query.  A query's chunks double without a cap, so one query whose merge a long run of
 *            tombstones or superseded versions holds back can stage past the budget, up to about twice that run.
 *   Errors.  DBEEL_ERR_CAPACITY as dbeel_get_values: the rows filled, out->data_len / index_len = the sizes needed, nothing
 *            written.  DBEEL_ERR_INVALID_ARG for a null pointer, n_ranges == 0, a limit of 0 or above
 *            DBEEL_RANGE_LIMIT_MAX, a sum of limits >= 2^32 - 16, or a flag other than DBEEL_RANGE_KEEP_TOMBSTONES.  A
 *            callback's nonzero return comes back unchanged; the reader, the engine and an attached page cache stay usable
 *            after every error.  DBEEL_ERR_BUSY while another call runs.  out->bloom is not used.
 * dbeel_last_stats: input_bytes = every byte read through the callback in this call, entries_in = index records staged,
 * output_bytes / entries_out = what was returned, partitions = merge rounds run, summed over groups; kernel_launches and
 * gather_bytes summed over the rounds, ms_total from the first round to the last output copy. */
#define DBEEL_RANGE_LIMIT_MAX 65536u
#define DBEEL_RANGE_MORE 0x1u     /* the range holds more entries than were returned */
#define DBEEL_RANGE_STOPPED 0x2u  /* stop says where; no entries */
#define DBEEL_RANGE_UNSORTED 0x4u /* stop.table's records read for it do not strictly ascend; stop.record = the first one
                                     not above its predecessor; no entries */
typedef struct dbeel_range_row {
    uint64_t first;       /* entry number in out of the query's first entry */
    uint32_t count;       /* entries returned */
    uint32_t flags;       /* DBEEL_RANGE_* */
    dbeel_scan_stop stop; /* {-1, DBEEL_SCAN_STOP_NONE, 0} unless STOPPED / UNSORTED */
} dbeel_range_row;
int dbeel_reader_get_ranges(dbeel_reader *r, const dbeel_key_ranges *ranges, uint32_t n_ranges, const uint32_t *limits,
                            uint32_t flags, dbeel_out *out, dbeel_range_row *rows);

/* Range reads from the end, batched: the LAST entries of many key ranges, in descending key order (the last page of a
 * listing, the previous page from a cursor, the newest events when keys end in a timestamp).  Arguments, ranges, limits
 * and flags as dbeel_reader_get_ranges; G_q as there (destination 0 of dbeel_reader_get_range for range q alone, in
 * ascending key order).
 *   Clean.   A query whose range makes that call return no stop and not DBEEL_ERR_UNSORTED_RUN gets the last
 *            min(limits[q], |G_q|) entries of G_q, in descending key order, byte for byte; DBEEL_RANGE_MORE is set iff
 *            |G_q| > limits[q].  A query with start >= end gets count 0, reads nothing and is never stopped, except by an
 *            empty table.
 *   Output.  Entries packed as dbeel_get_values packs them: query order, DESCENDING keys within a query, bytes as stored;
 *            the .index offsets start at 0 in out->data, key_size = 8 + klen, out->items_written = the total.  Row q's
 *            entries are entry numbers [first, first + count).  A caller asks for the previous page with end = the last
 *            (smallest) key returned: end is exclusive, so no key suffix is needed.
 *   Stops.   As dbeel_reader_get_ranges: a failed bound search or a table with no index record gives DBEEL_RANGE_STOPPED
 *            with that stop, and nothing is read for the query's records.
 *   Damage.  Only a suffix of every span is read.  Let A'_q be the merge, under G_q's rule, of every table's span records
 *            for q, each cut just above the first record met walking down from seek_t(end) - 1 that fails dbeel_scan's
 *            decode (ERR / PANIC as the scan classifies it) or whose key is not strictly below the key of the record
 *            after it.  The row is then either the last min(limit, |A'_q|) entries of A'_q in descending order (MORE iff
 *            |A'_q| > limit), or DBEEL_RANGE_STOPPED with stop = (table, ERR / PANIC, record) of a record that fails the
 *            decode, or DBEEL_RANGE_UNSORTED with stop = (table, DBEEL_SCAN_STOP_NONE, r) of a record r whose key is not
 *            below record r + 1's.  The last record of every non-empty span is always read.  One query's damage never
 *            changes another query's row.
 *   Reads.   The bound searches of dbeel_reader_get_ranges; per query and table, index records from seek_t(end) - 1
 *            downward, never below seek_t(start), in chunks that end at seek_t(end) and double for the tables that hold
 *            back the merge; the .data windows of exactly the records staged, each never wider than its records.  Leaf
 *            slices, staged index slices and windows go through an attached page cache.  Nothing else is read.
 *   Memory, Errors and dbeel_last_stats as dbeel_reader_get_ranges (DBEEL_RANGE_UNSORTED's stop.record here is the
 *            record not below its successor).  A flag other than DBEEL_RANGE_KEEP_TOMBSTONES is DBEEL_ERR_INVALID_ARG. */
int dbeel_reader_get_ranges_reverse(dbeel_reader *r, const dbeel_key_ranges *ranges, uint32_t n_ranges, const uint32_t *limits,
                                    uint32_t flags, dbeel_out *out, dbeel_range_row *rows);

/* Range reads across readers: the limited range-read batches of many readers of one engine in one call (a node whose
 * shards each have a page of a listing waiting, next pages and previous pages mixed), so that they share the bound
 * searches and the merge rounds instead of paying them once per reader.  Batch b asks
 * dbeel_reader_get_ranges(reader, &ranges, n_ranges, limits, flags, ...) when reverse is 0 and
 * dbeel_reader_get_ranges_reverse(...) when it is 1; a batch of n_ranges 0 asks nothing.
 * Result: exactly those solo calls for b = 0, 1, ... in order, concatenated.  rows has sum(n_ranges) rows in batch order;
 * each row's count, flags and stop are its solo row's (stop.table is a position in that batch's own reader's tables), and
 * its first is the solo row's first plus the entries of the batches before it.  out is the solo outputs appended: batch
 * b's .index offsets are shifted by the .data bytes before it; items_written is the total.  One batch's damage, stops,
 * empty tables or tombstone runs never change another batch's rows, also for two batches on the same reader, in the same
 * or opposite directions.
 * Reads: the bound searches of all batches run together: each batch's bounds are cut into its solo call's seek batches
 * (the same depth and cache decisions per table), and seek batches of consecutive batches share one search while they fit
 * the partition budget.  The merge rounds run the live queries of all batches together: each batch's groups are its solo
 * call's, packed whole in batch order while they fit the budget and each page cache's capacity.  A query's chunks,
 * doubling and finish test depend on its own state only, so its row is its solo row in any group.  Every read goes through
 * the pair's own reader's io->read and page cache, and lies inside what the solo calls, made in batch order on readers in
 * the same state, read for that table and file kind.  With no page cache, input_bytes is at most the sum of the solo
 * calls'.
 * Errors leave every reader, the engine and every page cache usable: DBEEL_ERR_INVALID_ARG for null batches / out / rows,
 * n_batches of 0 or above DBEEL_MAX_READER_BATCHES, a null reader or a reader of another engine, a null key_offsets or
 * limits in a batch with ranges, key_offsets that decrease, null keys with key bytes, a limit of 0 or above
 * DBEEL_RANGE_LIMIT_MAX, a flag other than DBEEL_RANGE_KEEP_TOMBSTONES, reverse above 1 or nonzero reserved, or a sum of
 * all limits >= 2^32 - 16; DBEEL_ERR_CAPACITY as dbeel_reader_get_ranges (every row filled, out->data_len / index_len =
 * the sizes the whole call needs, nothing written); a callback's nonzero return unchanged; DBEEL_ERR_BUSY while another
 * call runs on the engine.
 * dbeel_last_stats: input_bytes = every byte read through every reader's callback, entries_in = index records staged,
 * partitions = merge rounds run, kernel_launches and gather_bytes summed, entries_out / output_bytes = what was returned. */
typedef struct dbeel_range_batch {
    dbeel_reader *reader;
    dbeel_key_ranges ranges; /* 2 * n_ranges + 1 key offsets, as dbeel_reader_get_ranges */
    const uint32_t *limits;  /* n_ranges limits */
    uint32_t n_ranges;       /* 0 allowed: the batch asks nothing */
    uint32_t flags;          /* DBEEL_RANGE_KEEP_TOMBSTONES only */
    uint32_t reverse;        /* 0: dbeel_reader_get_ranges, 1: dbeel_reader_get_ranges_reverse */
    uint32_t reserved;       /* 0 */
} dbeel_range_batch;
int dbeel_readers_get_ranges(dbeel_engine *e, const dbeel_range_batch *batches, uint32_t n_batches, dbeel_out *out,
                             dbeel_range_row *rows);
void dbeel_reader_close(dbeel_reader *r);

/* Page cache for readers: the reference reads every .data / .index byte of a lookup or seek through a per-shard cache of
 * 4096-byte pages (CachedFileReader::read_at_into over PartitionPageCache, cached_file_reader.rs:28-79); this one keeps such
 * pages on the device, across batches and across the readers attached to it.
 *   - dbeel_page_cache_create: bytes / 4096 page slots in one device allocation on the engine's device, made now; the page
 *     table lives on the host, and no other device memory is taken.  Fewer than one slot is DBEEL_ERR_INVALID_ARG, a failed
 *     allocation DBEEL_ERR_NOMEM.
 *   - A page is the 4096 bytes at a page-aligned offset of one reader table's .data or .index; a file's last page holds only
 *     the bytes up to the file's length (never anything past EOF).  It is keyed by (table, file kind, page), where a table
 *     is what a tree's readers share (a reader opened after a flush hits on every table it shares with the reader before
 *     it), and a table that is gone is never hit again: its pages age out.
 *   - Contract: a reader's table files do not change while it is open (SSTables are immutable; cached fences assume it too).
 *   - dbeel_reader_attach_page_cache(r, c) makes r read through c from its next call; NULL detaches.  A cache of another
 *     engine is DBEEL_ERR_INVALID_ARG.  Any number of readers may share one cache.
 *   - Through the cache go the leaf .index slices and .data windows of dbeel_reader_get_values and the entries of its hits
 *     at fences, and the leaf slices and windows of dbeel_reader_scan's seeks (DBEEL_SCAN_KEY).  Resident pages are copied
 *     on the device; the missing ones are read through io.read as page-aligned ranges clipped to the file's length (the
 *     consecutive missing pages of a file as one read, in pieces of at most 8 MiB), and become resident only once their
 *     read has returned 0.  Eviction is CLOCK (second chance); the pages one step of a call needs are never evicted by it.
 *     A step that needs more pages than the cache has slots (a leaf larger than the cache) reads uncached.
 *   - Not through the cache: fence loads and per-call fences (a reader keeps its fences itself), hash scans, and the span
 *     partitions of key scans, which stream whole ranges once and would evict the point-read working set.
 *   - A cached reader returns exactly what it returns uncached (rows and flags, out, items_written, DBEEL_ERR_CAPACITY with
 *     the sizes needed, stops, callback codes unchanged); only what goes through the callback changes, and
 *     dbeel_last_stats' input_bytes still counts it.  After a callback error the cache holds only good pages, and both the
 *     reader and the cache stay usable.
 *   - dbeel_page_cache_stats: capacity / resident in pages; hits, misses and evictions in pages since create.
 *   - dbeel_page_cache_destroy detaches the cache from every reader that has it (they go on uncached);
 *     dbeel_engine_destroy destroys the caches still open.  Create, attach and stats take the engine as every entry point
 *     does (DBEEL_ERR_BUSY while another call runs). */
typedef struct dbeel_page_cache dbeel_page_cache;
/* a struct tag only, as POSIX's struct stat beside stat(): the function takes the plain name */
struct dbeel_page_cache_stats {
    uint64_t capacity_pages, resident_pages;
    uint64_t hits, misses, evictions; /* pages, since create */
};
int dbeel_page_cache_create(dbeel_engine *e, uint64_t bytes, dbeel_page_cache **out);
void dbeel_page_cache_destroy(dbeel_page_cache *c);
int dbeel_reader_attach_page_cache(dbeel_reader *r, dbeel_page_cache *c /* NULL detaches */);
int dbeel_page_cache_stats(const dbeel_page_cache *c, struct dbeel_page_cache_stats *out);

/* ---- N4: write-ahead-log replay + flush ------------------------------------------------------------------------
 * Replaces LSMTree::read_memtable_from_wal_file (lsm_tree.rs:552-574) followed by flush_memtable_to_disk, i.e. the
 * recovery of an unflushed memtable in open_or_create_ex (:478-513).  `wal` is the whole `.memtable` file: bincode
 * Entries at 4096-aligned offsets, each padded to `size + 4096 - size % 4096` (:740-744).  Replay rules kept:
 * the cursor moves to the first page boundary strictly after every record; an entry whose timestamp does not
 * deserialize is skipped; a record that runs past the end of the file ends the replay; an all-zero page is the entry
 * (key = [], data = [], timestamp = 0).  `capacity` is the memtable's (DEFAULT_TREE_CAPACITY, mod.rs:18): more distinct
 * keys than that fail the reference's replay with ReachedCapacity -> DBEEL_ERR_TREE_FULL.  out->data / out->index
 * receive the SSTable; caps: the sum of the logged entries' sizes (<= wal_len) and 16 bytes per logged entry
 * (<= 16 * ceil(wal_len / 4096)).  No bloom (lsm_tree.rs:908). */
int dbeel_wal_flush(dbeel_engine *e, const void *wal, uint64_t wal_len, uint32_t capacity, dbeel_out *out);
int dbeel_wal_flush_device(dbeel_engine *e, const void *wal, uint64_t wal_len, uint32_t capacity, dbeel_out *out);

/* Bloom::new_for_fp_rate arithmetic (bloomfilter 1.0.12). */
uint64_t dbeel_bloom_bitmap_bytes(uint64_t items, double fp);
uint32_t dbeel_bloom_k_num(uint64_t bitmap_bits, uint64_t items);
uint64_t dbeel_bloom_file_size(uint64_t items, double fp);

/* Pinned host memory for the host entry points (optional; any host pointer is accepted). */
void *dbeel_host_alloc(uint64_t bytes);
void dbeel_host_free(void *p);

int dbeel_last_stats(const dbeel_engine *e, dbeel_stats *out);
const char *dbeel_last_error(const dbeel_engine *e);
const char *dbeel_strerror(int code);
int dbeel_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DBEEL_COMPACT_H */
