/*
 * get_values_oracle.c -- CPU restatement of LSMTree::get_entry's SSTable loop with the entry it returns (test
 * infrastructure).
 *
 * It is compiled together with oracle/dbeel_oracle.c, whose orc_get_many (the search, lsm_tree.rs:605-670, 686-719),
 * timestamp check and EntryWriter it reuses, and restates (paths relative to the reference, tontinton/dbeel):
 *
 *   binary_search's decode of a hit ... src/storage_engine/lsm_tree.rs:628-651: read_at(offset, key_size) deserializes
 *                                       to the key, read_at(offset + key_size, full_size - key_size) to one EntryValue
 *   bincode options ................... src/utils/bincode.rs:8-16 (fixint, reject_trailing_bytes)
 *   EntryValue's timestamp ............ src/utils/timestamp_nanos.rs:15-24
 *
 * The answered entries are written the way EntryWriter writes records (entry_writer.rs:71-98), in query order.
 */
#include "../oracle/dbeel_oracle.c"

#define ORC_LOOKUP_BAD_ENTRY 0x40000000u

/* does the hit at index record `record` of `t` decode for a query key of klen bytes?  On success *e points INTO the
 * table (key, value) -- nothing is allocated */
static int hit_decodes(const orc_run *t, uint64_t record, uint64_t klen, orc_entry *e) {
    const uint8_t *rec = t->index + record * INDEX_ENTRY_SIZE;
    const uint64_t offset = rd_u64(rec);
    const uint64_t key_size = rd_u32(rec + 8), full_size = rd_u32(rec + 12);
    /* the key frame: u64 length + bytes, nothing after (the search already compared the bytes) */
    if (key_size != 8 + klen) return 0;
    /* the value frame: u64 dlen | data | i128 timestamp, exactly full_size - key_size bytes, all inside .data */
    if (full_size < key_size || offset > t->data_len || full_size > t->data_len - offset) return 0;
    const uint8_t *v = t->data + offset + key_size;
    const uint64_t n = full_size - key_size;
    if (n < 8) return 0;
    const uint64_t dlen = rd_u64(v);
    if (dlen > n - 8 || n - 8 - dlen != 16) return 0;
    __int128 ts;
    memcpy(&ts, v + 8 + dlen, 16);
    if (!timestamp_decodes(ts)) return 0;
    e->key = (uint8_t *)t->data + offset + 8;
    e->klen = klen;
    e->val = (uint8_t *)v + 8;
    e->dlen = dlen;
    e->ts = ts;
    return 1;
}

/* orc_get_many's rows, then per hit the decode above: a hit that does not decode gets ORC_LOOKUP_BAD_ENTRY (get_entry's
 * `binary_search(..).await?` returns Err) and no entry; every other hit's entry goes through EntryWriter into *out. */
int orc_get_values(const orc_run *tables, const uint8_t *const *blooms, const uint64_t *bloom_lens, uint32_t n_tables,
                   const uint8_t *keys, const uint64_t *key_off, uint64_t n_keys, int32_t *out_table, uint64_t *out_record,
                   uint32_t *out_rejects, orc_out *out) {
    orc_get_many(tables, blooms, bloom_lens, n_tables, keys, key_off, n_keys, out_table, out_record, out_rejects);
    entry_writer *w = (entry_writer *)malloc(sizeof *w);
    if (!w || !writer_init(w, out, 0)) { free(w); return ORC_ERR_NOMEM; }
    int rc = ORC_OK;
    for (uint64_t q = 0; q < n_keys && rc == ORC_OK; q++) {
        if (out_table[q] < 0) continue;
        orc_entry e;
        if (!hit_decodes(&tables[out_table[q]], out_record[q], key_off[q + 1] - key_off[q], &e)) {
            out_rejects[q] |= ORC_LOOKUP_BAD_ENTRY;
            continue;
        }
        rc = writer_write(w, &e);
    }
    writer_close(w);
    free(w);
    out->items_written = out->index_len / INDEX_ENTRY_SIZE;
    return rc;
}
