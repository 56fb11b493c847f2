/*
 * scan_oracle.c -- CPU restatement of LSMTree::iter_filter over a tree's SSTables (test infrastructure).
 *
 * It is compiled together with oracle/dbeel_oracle.c, whose entry decoder (entry_decode), murmur3_32 and EntryWriter it
 * reuses, and restates (paths relative to the reference, tontinton/dbeel):
 *
 *   AsyncIter::read_one .... src/storage_engine/lsm_tree.rs:210-281 (tables oldest first, sizes from :453)
 *   CachedFileReader ....... src/storage_engine/cached_file_reader.rs:60-90 (read_at panics: size 0, past the end)
 *   between_cmp ............ src/tasks/migration.rs:54-60, destination = first range (:97-104)
 *   key-range filter ....... lsm_tree.rs:1363-1397 (start <= key < end, Vec<u8> order)
 *
 * Every destination's entries are written the way EntryWriter writes records (entry_writer.rs:71-98).
 */
#include "../oracle/dbeel_oracle.c"

#define ORC_SCAN_STOP_NONE 0u
#define ORC_SCAN_STOP_ERR 1u
#define ORC_SCAN_STOP_PANIC 2u

int orc_between_cmp(uint32_t hash, uint32_t start, uint32_t end) {
    if (end < start) {
        return hash < start || hash >= end; /* hash.cmp(start) == Less || hash.cmp(end) != Less */
    } else {
        return hash >= start && hash < end; /* hash.cmp(start) != Less && hash.cmp(end) == Less */
    }
}

/* kind 0: hash_ranges[2 n_ranges]; kind 1: range d = [keys[key_off[2d]..key_off[2d+1]), keys[key_off[2d+1]..key_off[2d+2])).
 * outs[d] receives destination d's SSTable.  Returns ORC_OK or an orc error code; *stop_* say where the iterator ended. */
int orc_scan(const orc_run *tables, uint32_t n_tables, uint32_t kind, const uint32_t *hash_ranges, const uint8_t *keys,
             const uint64_t *key_off, uint32_t n_ranges, orc_out *outs, int32_t *stop_table, uint32_t *stop_reason,
             uint64_t *stop_record) {
    *stop_table = -1;
    *stop_reason = ORC_SCAN_STOP_NONE;
    *stop_record = 0;
    entry_writer *w = (entry_writer *)calloc(n_ranges ? n_ranges : 1, sizeof(entry_writer));
    if (!w) return ORC_ERR_NOMEM;
    for (uint32_t d = 0; d < n_ranges; d++) writer_init(&w[d], &outs[d], 0);
    int rc = ORC_OK;
    for (uint32_t t = 0; t < n_tables && rc == ORC_OK; t++) {
        const orc_run *tb = &tables[t];
        const uint64_t index_file_size = tb->index_len / INDEX_ENTRY_SIZE * INDEX_ENTRY_SIZE; /* sstable.size * 16 */
        uint64_t index_offset = 0;
        for (;;) {
            uint32_t reason = ORC_SCAN_STOP_NONE;
            /* index_file.read_at_into(index_offset, 16): past the end of the file -> panic */
            if (index_offset + INDEX_ENTRY_SIZE > tb->index_len) {
                reason = ORC_SCAN_STOP_PANIC;
            } else {
                const uint8_t *rec = tb->index + index_offset;
                const uint64_t offset = rd_u64(rec);
                const uint32_t full_size = rd_u32(rec + 12); /* key_size (rec + 8) is not read */
                orc_entry e;
                if (full_size == 0 || offset > tb->data_len || full_size > tb->data_len - offset) {
                    reason = ORC_SCAN_STOP_PANIC; /* assert_ne!(size, 0) / slice out of range */
                } else if (!entry_decode(tb->data + offset, full_size, &e)) {
                    reason = ORC_SCAN_STOP_ERR;
                } else {
                    int dest = -1;
                    if (kind == 0) {
                        const uint32_t h = orc_murmur3_32(e.key, e.klen, 0);
                        for (uint32_t d = 0; d < n_ranges && dest < 0; d++)
                            if (orc_between_cmp(h, hash_ranges[2 * d], hash_ranges[2 * d + 1])) dest = (int)d;
                    } else {
                        for (uint32_t d = 0; d < n_ranges && dest < 0; d++) {
                            const uint8_t *s = keys + key_off[2 * d], *en = keys + key_off[2 * d + 1];
                            const uint64_t sl = key_off[2 * d + 1] - key_off[2 * d], el = key_off[2 * d + 2] - key_off[2 * d + 1];
                            if (key_cmp(s, sl, e.key, e.klen) <= 0 && key_cmp(e.key, e.klen, en, el) < 0) dest = (int)d;
                        }
                    }
                    if (dest >= 0) rc = writer_write(&w[dest], &e);
                    entry_free(&e);
                }
            }
            if (reason != ORC_SCAN_STOP_NONE) {
                *stop_table = (int32_t)t;
                *stop_reason = reason;
                *stop_record = index_offset / INDEX_ENTRY_SIZE;
                goto done;
            }
            if (rc != ORC_OK) break;
            index_offset += INDEX_ENTRY_SIZE;
            if (index_offset >= index_file_size) break;
        }
    }
done:
    for (uint32_t d = 0; d < n_ranges; d++) {
        writer_close(&w[d]);
        outs[d].items_written = outs[d].index_len / INDEX_ENTRY_SIZE;
    }
    free(w);
    return rc;
}
