// reader_tables.h -- the engine's side of readers (dbeel_reader_*) as the tree's shared cache entries use it (internal to
// the library: dbeel_compact.cu defines it, host/lsm_tree_host.cc calls it).
//
// A reader table is one SSTable's device-resident part: its filter, uploaded when the table is created, and its fences,
// read the first time a batch in a mode reaches it.  Readers hold their tables by reference count, so several readers of
// one tree share the tables they have in common.
#pragma once
#include <memory>
#include <vector>

#include "../../../include/dbeel_compact.h"

struct dbeel_reader_table;

namespace dbeel {

using ReaderTableRef = std::shared_ptr<dbeel_reader_table>;

// t: lengths and the .bloom in host memory (.data / .index are ignored); the filter is validated and uploaded now.
int reader_table_create(dbeel_engine *e, const dbeel_table &t, ReaderTableRef *out);

// A reader over `tables` (oldest first) that reads .data / .index through `io`, holding `owner` (what io.ctx points at)
// until it is closed.
int reader_open_tables(dbeel_engine *e, std::vector<ReaderTableRef> tables, const dbeel_scan_io &io, uint64_t fence_bytes,
                       std::shared_ptr<void> owner, dbeel_reader **out);

} // namespace dbeel
