/*
 * dbeel_tree.h -- host-side mirror of the file protocol AROUND the GPU path, C ABI.
 *
 * The reference is Rust (compiled code) and no Rust toolchain exists here, so the host side
 * above the engine's C ABI is C++ (dbeel_b200/csrc/host/lsm_tree_host.cc), mirroring the
 * reference's own interface for this path -- same names, argument meaning, error behaviour:
 *
 *   dbeel_tree_open        <- LSMTree::open_or_create_ex: journal replay + SSTable discovery
 *                             (src/storage_engine/lsm_tree.rs:424-465)
 *   dbeel_tree_recover_wal <- the rest of open_or_create_ex: an unflushed memtable's log is replayed and flushed
 *                             (lsm_tree.rs:466-513, read_memtable_from_wal_file :552-574) through dbeel_wal_flush()
 *   dbeel_tree_compact     <- LSMTree::compact(indices_to_compact, output_index, keep_tombstones)
 *                             (lsm_tree.rs:950-1156): same files, same CompactionAction journal
 *                             (:73-77, :1078-1111), same renames / deletes; the merge core
 *                             (:1002-1076) is dbeel_compact()
 *   dbeel_tree_flush       <- LSMTree::flush's SSTable part (lsm_tree.rs:875-915): writes the
 *                             next even index through dbeel_flush(), no bloom
 *   dbeel_tree_sstables    <- LSMTree::sstable_indices_and_sizes (lsm_tree.rs:592-598)
 *   dbeel_tree_get_many    <- the SSTable loop of LSMTree::get_entry (lsm_tree.rs:686-719) through dbeel_get_many()
 *   dbeel_tree_get_values  <- the same with the entries (:674-723) through dbeel_get_values()
 *   dbeel_tree_scan        <- the SSTable part of LSMTree::iter_filter (lsm_tree.rs:133-282, :1183-1189) through dbeel_scan()
 *   dbeel_tree_scan_stream <- the same through dbeel_scan_stream(): the files are streamed, trees of any size
 *   dbeel_memtable_cut     <- RedBlackTree::set + active_memtable_full (rbtree_arena lib.rs:497-534,
 *                             lsm_tree.rs:600-603,757-765): how many arrivals fill one memtable
 *   dbeel_plan_compactions <- compact_tree's size-tiered picker (src/tasks/compaction.rs:35-102),
 *                             made deterministic (the reference enumerates a HashMap)
 */
#ifndef DBEEL_TREE_H
#define DBEEL_TREE_H

#include <stdint.h>

#include "dbeel_compact.h"

#ifdef __cplusplus
extern "C" {
#endif

#define DBEEL_ERR_IO 20        /* a filesystem call failed; dbeel_tree_last_error() has errno text */
#define DBEEL_ERR_NO_SSTABLE 21 /* an index in indices_to_compact has no .data/.index files */

typedef struct dbeel_tree dbeel_tree;

/* EntryWriter's page-cache write-through (src/storage_engine/entry_writer.rs:94-156): while it writes an SSTable the
 * reference mirrors both streams into the shard's page cache in 4 KiB pages keyed by ((FileTypeKind, files_index), page
 * address), the last page of each stream zero-padded at close().  dbeel_out_pages replays exactly those `set` calls -- same
 * pages, same order -- for an SSTable the engine produced (host buffers), so the Rust side can warm its PartitionPageCache
 * from the returned buffers.  Not on-disk state: skipping it can never serve stale bytes (the keys carry the fresh index). */
#define DBEEL_FILE_DATA 1u  /* FileTypeKind::Data  (mod.rs:36-42: Memtable, Data, Index, Bloom) */
#define DBEEL_FILE_INDEX 2u /* FileTypeKind::Index */
typedef void (*dbeel_page_sink)(void *ctx, uint32_t file_kind, uint64_t files_index, uint64_t address, const uint8_t *page /* 4096 bytes */);
int dbeel_out_pages(const void *data, uint64_t data_len, const void *index, uint64_t index_len, uint64_t files_index,
                    dbeel_page_sink sink, void *ctx);
/* A tree with a sink installed calls it for every SSTable dbeel_tree_compact / _compact_many / _flush / _recover_wal write. */
void dbeel_tree_set_page_sink(dbeel_tree *t, dbeel_page_sink sink, void *ctx);

int dbeel_tree_open(const char *dir, dbeel_engine *engine, uint64_t sstable_bloom_min_size, dbeel_tree **out);
void dbeel_tree_close(dbeel_tree *t);

/* (index, size = entries) of every SSTable, ascending by index.  Returns the count; fills up to cap. */
uint32_t dbeel_tree_sstables(const dbeel_tree *t, uint64_t *indices, uint64_t *sizes, uint32_t cap);
uint64_t dbeel_tree_write_sstable_index(const dbeel_tree *t); /* next even index a flush will use */

int dbeel_tree_compact(dbeel_tree *t, const uint64_t *indices_to_compact, uint32_t n, uint64_t output_index,
                       int keep_tombstones, const uint8_t *bloom_seed /* 32 bytes or NULL */);

/* compact_tree's loop (tasks/compaction.rs:82-101) in one go: all groups of a dbeel_plan_compactions() result (same
 * flattened layout) are merged by ONE dbeel_compact_many() call, then committed group by group exactly like
 * dbeel_tree_compact.  bloom_seeds: 32 bytes per group back to back, or NULL. */
int dbeel_tree_compact_many(dbeel_tree *t, const uint64_t *members, const uint32_t *group_start, uint32_t n_groups,
                            const uint64_t *output_index, const int32_t *keep_tombstones, const uint8_t *bloom_seeds);

/* Flush one memtable's arrivals (host buffers, arrival order) to the next even index. */
int dbeel_tree_flush(dbeel_tree *t, const dbeel_run *batch, uint64_t *written_index, uint64_t *items_written);

/* The SSTable loop of LSMTree::get_entry (lsm_tree.rs:686-719) for a batch of keys, over the tree's files (each table
 * with its .bloom if the file exists): results[i].table is a position in dbeel_tree_sstables() order.  Keys / modes /
 * rows as in dbeel_get_many.  The memtable look-ups in front of it (:677-684) are the caller's. */
int dbeel_tree_get_many(dbeel_tree *t, const void *keys, const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode,
                        dbeel_lookup_result *results);

/* dbeel_tree_get_many with the entries: the tree's files read whole as there, then dbeel_get_values() (rows, output,
 * caps and DBEEL_ERR_CAPACITY as described there).  out is host memory. */
int dbeel_tree_get_values(dbeel_tree *t, const void *keys, const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode,
                          dbeel_out *out, dbeel_lookup_result *results);

/* dbeel_tree_get_values with the files left on disk (dbeel_get_values_stream): each .bloom is read whole, as the reference
 * does when it opens a table; .data and .index are pread only where the batch's searches reach, so a tree larger than device
 * or host memory answers too.  Rows, output, caps and DBEEL_ERR_CAPACITY equal dbeel_tree_get_values'.  out is host memory. */
int dbeel_tree_get_values_stream(dbeel_tree *t, const void *keys, const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode,
                                 dbeel_out *out, dbeel_lookup_result *results);

/* A reader (dbeel_reader_open) over a snapshot of the tree's SSTables: dbeel_tree_sstables() at open, the `sstables` clone
 * get_entry and AsyncIter take (lsm_tree.rs:177, 686).  dbeel_reader_get_values on it returns what
 * dbeel_tree_get_values_stream returned at open, with results[i].table a position in the snapshot; close it with
 * dbeel_reader_close.  The reader holds every table's .data / .index descriptors until it is closed, so a later compaction
 * that unlinks its inputs does not disturb it (as the reference promises its iterators, :175-176).
 * The tree keeps one entry per SSTable (device filter, fences per mode, descriptors), shared by reference count between
 * the readers that include the table: a reader opened after a flush or a compaction loads only the tables no live entry
 * has, and a table it shares keeps the fence depth it was loaded with (its fences count against fence_bytes first).  An
 * entry is dropped when no reader holds it and its table has left the tree; dbeel_tree_close drops the tree's entries
 * (open readers keep theirs until they are closed).
 * A device page cache (dbeel_page_cache_create, dbeel_reader_attach_page_cache) keys its pages by that shared entry, so a
 * reader opened after a flush and attached to the same cache hits on every table it shares with the readers before it.
 * The tree's own page sink (dbeel_tree_set_page_sink) is a separate, host-side mirror and does not fill it. */
int dbeel_tree_reader_open(dbeel_tree *t, uint64_t fence_bytes, dbeel_reader **out);

/* The SSTable part of LSMTree::iter_filter over the tree's files: every table's .data / .index in dbeel_tree_sstables()
 * order (oldest first, the iterator's order) through one dbeel_scan().  kind / ranges / results / stop as in dbeel_scan;
 * out holds host buffers (caps: the sums of the tables' .data and .index file sizes).  stop->table is a position in
 * dbeel_tree_sstables() order.  The memtables the iterator emits after the tables (:155-173) are the caller's. */
int dbeel_tree_scan(dbeel_tree *t, uint32_t kind, const void *ranges, uint32_t n_ranges, dbeel_out *out,
                    dbeel_job_result *results, dbeel_scan_stop *stop);

/* The same scan with the files streamed through the engine (dbeel_scan_stream): the tables are pread in pieces, nothing is
 * held whole in memory, so a tree larger than device or host memory scans too (migration of a shard's whole tree).  Every
 * destination's output goes to `write` (dbeel_scan_io.write: destination d's .data / .index from offset 0, pieces in any
 * order, from several threads); its error code comes back unchanged.  results / stop as dbeel_scan_stream. */
int dbeel_tree_scan_stream(dbeel_tree *t, uint32_t kind, const void *ranges, uint32_t n_ranges,
                           int (*write)(void *ctx, uint32_t dest, uint32_t kind, uint64_t offset, const void *src, uint64_t len),
                           void *ctx, dbeel_job_result *results, dbeel_scan_stop *stop);

/* WAL recovery step of open_or_create_ex.  0 logs: *wal_file_index = 0; 1 log: its index; 2 logs: the older one is
 * replayed (memtable of `tree_capacity` entries, DBEEL_ERR_TREE_FULL like the reference's ReachedCapacity), flushed
 * to `<newer index>.data / .index` exactly as the reference does, and removed; more than 2: error (the reference
 * panics).  *items_written = entries of the recovered SSTable (0 if nothing was recovered). */
int dbeel_tree_recover_wal(dbeel_tree *t, uint32_t tree_capacity, uint64_t *wal_file_index, uint64_t *items_written);

const char *dbeel_tree_last_error(const dbeel_tree *t);

/* Number of arrivals, starting at `first_record`, that a memtable of `capacity` distinct keys
 * absorbs before it is full (the insert that fills it included); the rest of the batch if it
 * never fills. */
uint64_t dbeel_memtable_cut(const dbeel_run *batch, uint64_t first_record, uint32_t capacity);

/* compact_tree's picker.  In: n SSTables (index, size).  Out: groups to compact, flattened:
 * group g covers members[group_start[g] .. group_start[g+1]) (SSTable indices, in the order they
 * must be passed as indices_to_compact), writes output_index[g], with keep_tombstones[g].
 * Groups are ordered largest tables first, so only the final level drops tombstones
 * (compaction.rs:91-92).  Returns the number of groups (<= n / 2). */
uint32_t dbeel_plan_compactions(const uint64_t *indices, const uint64_t *sizes, uint32_t n,
                                uint32_t compaction_factor, uint64_t *members, uint32_t *group_start,
                                uint64_t *output_index, int32_t *keep_tombstones);

#ifdef __cplusplus
}
#endif
#endif /* DBEEL_TREE_H */
