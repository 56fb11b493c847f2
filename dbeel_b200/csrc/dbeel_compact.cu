// dbeel_compact.cu -- engine + C ABI (include/dbeel_compact.h) over the kernels in kernels.cuh.
//
// One engine = one GPU + one stream + a grow-only device workspace.  A compaction job is a
// fixed sequence of kernel launches with no host round trip in between; the only host sync
// is the final read-back of the 300-byte control block (output lengths, flags).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <deque>
#include <memory>
#include <new>
#include <thread>
#include <string>
#include <vector>

#include "../../include/dbeel_compact.h"
#include "kernels.cuh"
#include "merge_final.cuh"
#include "merge_range.cuh"
#include "range_limit.cuh"
#include "gather_h.cuh"
#include "lookup.cuh"
#include "lookup_stream.cuh"
#include "route.cuh"
#include "scan.cuh"
#include "wal.cuh"
#include "host/page_cache.h"
#include "host/reader_tables.h"
#include "host/scan_plan.h"
#include "host/stream_pump.h"

using namespace dbeel;

namespace {

constexpr uint64_t kAlign = 256;
inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

// the offset of the next b bytes of a workspace being laid out at *off, each piece 256-byte aligned
uint64_t carve_ws(uint64_t *off, uint64_t b) {
    const uint64_t o = *off;
    *off = align_up(*off + b, kAlign);
    return o;
}

enum { EV_START = 0, EV_EXTRACT, EV_MERGE, EV_RESOLVE, EV_GATHER, EV_H2D0, EV_H2D1, EV_D2H0, EV_D2H1, EV_COUNT };

} // namespace

struct dbeel_engine {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[EV_COUNT] = {};
    // device workspace (grow-only)
    uint8_t *ws = nullptr;
    uint64_t ws_cap = 0;
    // device staging for the host entry points (grow-only)
    uint8_t *stage_in = nullptr, *stage_out = nullptr;
    uint64_t stage_in_cap = 0, stage_out_cap = 0;
    // pipelined host path: second staging pair, copy streams, shared bloom buffer
    uint8_t *stage_in2 = nullptr, *stage_out2 = nullptr, *bloom_dev = nullptr;
    uint64_t stage_in2_cap = 0, stage_out2_cap = 0, bloom_dev_cap = 0;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    cudaEvent_t ev_h2d[2] = {}, ev_comp[2] = {}, ev_d2h[2] = {};
    int pipeline = 1;                   // DBEEL_PIPELINE: 0 = single-shot host path
    uint64_t pipeline_min_bytes = 64ull << 20;
    uint64_t partition_bytes = 256ull << 20; // DBEEL_PARTITION_MB
    int partition_taper = 1;                 // DBEEL_PARTITION_TAPER: small first / last partitions (A/B switch)
    // streaming host path (dbeel_compact_stream): pinned rings the file bytes pass through, the runs' .index files, the filter
    // on its way out (grow-only, page-locked)
    uint8_t *ring_in = nullptr, *ring_out = nullptr, *pin_index = nullptr, *pin_bloom = nullptr;
    uint64_t ring_in_cap = 0, ring_out_cap = 0, pin_index_cap = 0, pin_bloom_cap = 0;
    int stream_ring = 3;                     // DBEEL_STREAM_RING: slots per ring (>= 2)
    // pinned host block: job header going down, control block coming back
    uint8_t *wal_ws = nullptr; // WAL replay: doubling tables + the arrival index (grow-only)
    uint64_t wal_ws_cap = 0;
    uint8_t *route_ws = nullptr; // shard routing: owners, block histograms, totals (grow-only)
    uint64_t route_ws_cap = 0;
    uint8_t *pin = nullptr;
    uint8_t *pin_dev = nullptr; // the same block as the GPU sees it (mapped: kernels read the header / write the control block)
    uint64_t pin_cap = 0;
    dbeel_stats stats = {};
    std::string err;
    std::atomic<bool> busy{false}; // a call holds the engine (Claim)
    std::vector<dbeel_reader *> readers; // open readers (dbeel_reader_open, dbeel_tree_reader_open): closed with the engine
    std::vector<dbeel_page_cache *> page_caches; // open page caches (dbeel_page_cache_create): destroyed with the engine
    // asynchronous jobs (dbeel_compact_submit)
    std::thread worker;
    std::atomic<int> async_state{0}; // 0 idle, 1 running, 2 finished (status in async_status)
    int async_status = 0;
    std::vector<dbeel_run> async_runs;
    dbeel_compact_opts async_opts = {};
    uint8_t async_seed[32] = {};
    int sm_count = 0; // multiProcessorCount of the device, set at engine creation
    int narrow_loads = 1;       // DBEEL_NARROW: .L2::64B loads for random accesses in extract / resolve (A/B switch)
    int fused_final = 1;        // DBEEL_FUSED_FINAL: 1 = last merge level + resolve + offsets scan + .index writes in one persistent kernel
                                // (k_merge_final, single compactions; the default: on an H100 it takes a cfg2 job from 5.91 ms with the five
                                // kernels to 3.96 ms, DESIGN.md section 7), 0 = the five kernels
    int fin_ctas_per_sm = 0;    // co-resident k_merge_final CTAs per SM (occupancy query at engine creation): its chained scan needs them all resident
    int pdl = 0;                // DBEEL_PDL: 1 = the job's kernels are launched with programmatic stream serialization (griddepcontrol)
    int stage_events = 1;       // DBEEL_STAGE_EVENTS: 0 = no per-stage event records inside a job (stage_ms read 0)
    int extract_persist = 6;    // DBEEL_EXTRACT_PERSIST: > 0 = k_extract runs as that many CTAs per SM, each thread fetching the next step's index
                                // records while the current step's entry headers travel
};

namespace {

// the engine whose asynchronous job runs on this thread (dbeel_compact_submit's worker)
thread_local const dbeel_engine *t_job_engine = nullptr;

// From dbeel_compact_submit until dbeel_poll / dbeel_wait reaps the job, e->err and e->stats are the job's: every other call
// is refused with DBEEL_ERR_BUSY and touches neither (BUSY is an expected answer for a reactor that polls).
bool refused(const dbeel_engine *e) { return e->async_state.load(std::memory_order_acquire) != 0 && t_job_engine != e; }

int fail(dbeel_engine *e, int code, const char *what, cudaError_t ce = cudaSuccess) {
    if (e && refused(e)) return DBEEL_ERR_BUSY; // an argument check ahead of the Claim: the job's error text stays
    char buf[512];
    if (ce != cudaSuccess)
        snprintf(buf, sizeof buf, "%s: %s (%s)", what, cudaGetErrorName(ce), cudaGetErrorString(ce));
    else
        snprintf(buf, sizeof buf, "%s", what);
    if (e) e->err = buf;
    return code;
}

#define CU(call)                                                            \
    do {                                                                    \
        cudaError_t ce_ = (call);                                           \
        if (ce_ != cudaSuccess) return fail(e, DBEEL_ERR_CUDA, #call, ce_); \
    } while (0)

int ensure_device(dbeel_engine *e, uint8_t **buf, uint64_t *cap, uint64_t need) {
    if (need <= *cap) return DBEEL_OK;
    if (*buf) { cudaFree(*buf); *buf = nullptr; *cap = 0; }
    uint64_t want = align_up(need + need / 8, 1 << 20);
    cudaError_t ce = cudaMalloc(reinterpret_cast<void **>(buf), want);
    if (ce != cudaSuccess) {
        cudaGetLastError();
        want = align_up(need, 1 << 20);
        ce = cudaMalloc(reinterpret_cast<void **>(buf), want);
    }
    if (ce != cudaSuccess) { cudaGetLastError(); return fail(e, DBEEL_ERR_NOMEM, "cudaMalloc(workspace)", ce); }
    *cap = want;
    return DBEEL_OK;
}

// Taking the engine.  Every call that uses it holds a Claim from where it takes the engine until it returns: refused (rc =
// DBEEL_ERR_BUSY, nothing touched) while an asynchronous job is unreaped, "engine busy" while another call holds it.  A
// taken engine starts with no error text and zeroed stats, on its device.
class Claim {
  public:
    explicit Claim(dbeel_engine *e) {
        if (refused(e)) { rc = DBEEL_ERR_BUSY; return; }
        if (e->busy.exchange(true, std::memory_order_acquire)) { rc = fail(e, DBEEL_ERR_BUSY, "engine busy"); return; }
        e_ = e;
        e->err.clear();
        e->stats = dbeel_stats{};
        const cudaError_t ce = cudaSetDevice(e->device);
        if (ce != cudaSuccess) rc = fail(e, DBEEL_ERR_CUDA, "cudaSetDevice", ce);
    }
    ~Claim() { if (e_) e_->busy.store(false, std::memory_order_release); }
    Claim(const Claim &) = delete;
    Claim &operator=(const Claim &) = delete;
    int rc = DBEEL_OK;

  private:
    dbeel_engine *e_ = nullptr;
};

// Host staging of the entry points that take whole host buffers.  Every piece starts 256-byte aligned and has kStageSlack
// bytes behind it: the kernels load an entry's 16-byte head as two ld_u64_unaligned (aligned 8-byte words) without
// checking where the buffer ends, so a head that starts in a piece's last 16 bytes reads up to 23 bytes past them.
constexpr uint64_t kStageSlack = 32;

struct HostPiece {
    const void *src;
    uint64_t len;
    const uint8_t *dev; // set by stage_host
};

// Lays the pieces back to back into stage_in and enqueues their copies on the engine's stream.
int stage_host(dbeel_engine *e, std::vector<HostPiece> &pieces) {
    uint64_t need = 0;
    for (const HostPiece &p : pieces) need += align_up(p.len + kStageSlack, kAlign);
    if (const int rc = ensure_device(e, &e->stage_in, &e->stage_in_cap, need)) return rc;
    uint64_t pos = 0;
    for (HostPiece &p : pieces) {
        p.dev = e->stage_in + pos;
        if (p.len) CU(cudaMemcpyAsync(e->stage_in + pos, p.src, p.len, cudaMemcpyHostToDevice, e->stream));
        pos += align_up(p.len + kStageSlack, kAlign);
    }
    return DBEEL_OK;
}

// *dout = outputs of data / index / bloom bytes in stage_out (bloom 0: none), with those capacities, nothing written yet.
int stage_outputs(dbeel_engine *e, uint64_t data, uint64_t index, uint64_t bloom, dbeel_out *dout) {
    const uint64_t o_index = align_up(data + kStageSlack, kAlign), o_bloom = o_index + align_up(index + kStageSlack, kAlign);
    if (const int rc = ensure_device(e, &e->stage_out, &e->stage_out_cap, o_bloom + (bloom ? align_up(bloom + kStageSlack, kAlign) : 0)))
        return rc;
    *dout = dbeel_out{e->stage_out, data, 0, e->stage_out + o_index, index, 0, bloom ? e->stage_out + o_bloom : nullptr, bloom, 0, 0};
    return DBEEL_OK;
}

// Enqueues the copies of what was written into outputs from stage_outputs (the filter: bloom_len bytes) back to `out` and
// sets its lengths; the caller synchronizes.
int copy_back(dbeel_engine *e, const dbeel_out &dout, uint64_t bloom_len, dbeel_out *out) {
    cudaStream_t s = e->stream;
    if (dout.data_len) CU(cudaMemcpyAsync(out->data, dout.data, dout.data_len, cudaMemcpyDeviceToHost, s));
    if (dout.index_len) CU(cudaMemcpyAsync(out->index, dout.index, dout.index_len, cudaMemcpyDeviceToHost, s));
    if (bloom_len) CU(cudaMemcpyAsync(out->bloom, dout.bloom, bloom_len, cudaMemcpyDeviceToHost, s));
    out->data_len = dout.data_len;
    out->index_len = dout.index_len;
    out->bloom_len = bloom_len;
    out->items_written = dout.items_written;
    return DBEEL_OK;
}

int ensure_pinned(dbeel_engine *e, uint64_t need) {
    if (need <= e->pin_cap) return DBEEL_OK;
    if (e->pin) cudaFreeHost(e->pin);
    e->pin = nullptr;
    e->pin_dev = nullptr;
    e->pin_cap = 0;
    cudaError_t ce = cudaHostAlloc(reinterpret_cast<void **>(&e->pin), need, cudaHostAllocMapped);
    if (ce != cudaSuccess) { cudaGetLastError(); return fail(e, DBEEL_ERR_NOMEM, "cudaHostAlloc", ce); }
    ce = cudaHostGetDevicePointer(reinterpret_cast<void **>(&e->pin_dev), e->pin, 0);
    if (ce != cudaSuccess) { cudaGetLastError(); return fail(e, DBEEL_ERR_CUDA, "cudaHostGetDevicePointer", ce); }
    e->pin_cap = need;
    return DBEEL_OK;
}

// grow-only page-locked host buffer (the streaming path's rings)
int ensure_host(dbeel_engine *e, uint8_t **buf, uint64_t *cap, uint64_t need) {
    if (need <= *cap) return DBEEL_OK;
    if (*buf) { cudaFreeHost(*buf); *buf = nullptr; *cap = 0; }
    const uint64_t want = align_up(need + need / 8, 1 << 20);
    cudaError_t ce = cudaHostAlloc(reinterpret_cast<void **>(buf), want, cudaHostAllocDefault);
    if (ce != cudaSuccess) { cudaGetLastError(); *buf = nullptr; return fail(e, DBEEL_ERR_NOMEM, "cudaHostAlloc(stream ring)", ce); }
    *cap = want;
    return DBEEL_OK;
}

int stream_threads() {
    static const int n = [] {
        if (const char *v = getenv("DBEEL_IO_THREADS")) return std::max(1, atoi(v));
        const unsigned hw = std::thread::hardware_concurrency();
        return (int)std::min(8u, std::max(2u, hw / 8)); // readers and writers each (measured on the 128-thread box: 8 + 8 = 16 + 16, 32 + 32 loses)
    }();
    return n;
}

// n independent pieces of callback I/O over a few threads; the first nonzero return code wins
template <class F>
int parallel_pieces(size_t n, F fn) {
    std::atomic<size_t> next{0};
    std::atomic<int> err{0};
    auto work = [&]() {
        for (size_t k = next.fetch_add(1); k < n && !err.load(); k = next.fetch_add(1)) {
            const int rc = fn(k);
            if (rc) { int z = 0; err.compare_exchange_strong(z, rc); }
        }
    };
    const int nt = (int)std::min<size_t>((size_t)stream_threads(), n);
    std::vector<std::thread> pool;
    for (int i = 1; i < nt; i++) pool.emplace_back(work);
    work();
    for (auto &t : pool) t.join();
    return err.load();
}

// the copy streams and events of the pipelined host paths (created on first use)
int ensure_copy_streams(dbeel_engine *e) {
    if (e->s_h2d) return DBEEL_OK;
    CU(cudaStreamCreateWithFlags(&e->s_h2d, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&e->s_d2h, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) {
        CU(cudaEventCreateWithFlags(&e->ev_h2d[i], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&e->ev_comp[i], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&e->ev_d2h[i], cudaEventDisableTiming));
    }
    return DBEEL_OK;
}

void default_opts(dbeel_compact_opts *o) {
    o->keep_tombstones = 0;
    o->flags = 0;
    o->bloom_min_size = DBEEL_DEFAULT_BLOOM_MIN_SIZE;
    o->bloom_fp = DBEEL_DEFAULT_BLOOM_FP;
    o->bloom_seed = nullptr;
}

// Kernel launch with (optionally) the programmatic-stream-serialization attribute: the kernel may be scheduled while its
// predecessor in the stream drains; every kernel starts with griddepcontrol.wait, so stream order is kept (kernels.cuh).
template <typename... KArgs, typename... Args>
void launch_k(const dbeel_engine *e, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = e->pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

struct JobShape {
    uint64_t n_total = 0; // sum of index_len / 16
    uint64_t data_total = 0;
    uint64_t index_total = 0; // sum of index_len (raw)
    uint64_t bloom_file = 0;  // 0 = no bloom
    uint64_t bloom_bits = 0, bloom_words = 0;
    uint32_t bloom_k = 0;
};

int shape_of(const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *o, bool flush, JobShape *s) {
    for (uint32_t r = 0; r < n_runs; r++) {
        s->n_total += runs[r].index_len / DBEEL_INDEX_ENTRY_SIZE;
        s->data_total += runs[r].data_len;
        s->index_total += runs[r].index_len;
    }
    // lsm_tree.rs:1026-1034: sized for the INPUT entry count, enabled on input .data bytes
    if (!flush && s->n_total > 0 && s->data_total > o->bloom_min_size) {
        uint64_t bytes = dbeel_bloom_bitmap_bytes(s->n_total, o->bloom_fp);
        s->bloom_bits = bytes * 8;
        s->bloom_words = (s->bloom_bits + 31) / 32;
        s->bloom_k = dbeel_bloom_k_num(s->bloom_bits, s->n_total);
        s->bloom_file = 8 + 4 * s->bloom_words + 8 + 8 + 4 + 144;
    }
    return DBEEL_OK;
}

// Set when a job is one key-range partition of a larger compaction (host entry point, section "pipelined").
struct JobExtra {
    const uint64_t *off_base = nullptr; // [n_runs] .data offset of each run slice's first byte; data pointers are pre-biased
    uint64_t out_offset_base = 0;       // .data bytes the earlier partitions wrote
    bool external_bloom = false;        // the filter belongs to the whole compaction: set bits only
    BloomParams bloom = {};
    dbeel_flush_table *flush_table = nullptr; // flush-many: one row per batch (host memory), filled on success
    // compact-many: runs[] holds all jobs' runs back to back; job g = runs[job_first[g] .. job_first[g+1])
    uint32_t n_jobs = 0;
    const uint32_t *job_first = nullptr;     // [n_jobs + 1]
    const int32_t *job_keep = nullptr;       // [n_jobs] keep_tombstones
    const BloomParams *job_bloom = nullptr;  // [n_jobs] device-side filter of each job (words == null: none)
    dbeel_job_result *job_results = nullptr; // [n_jobs] filled on success (bloom_off / bloom_len are the caller's)
    bool sparse_offsets = false;        // WAL replay: the batch's .data is the log itself, records do not abut
    uint64_t data_bytes = 0;            // with sparse_offsets: sum of the records' sizes (the output bound)
};

// The whole device-resident job.  `runs` / `out` hold device pointers.
int run_job_device(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *o,
                   bool flush, dbeel_out *out, const JobExtra *extra = nullptr) {
    JobShape sh;
    shape_of(runs, n_runs, o, flush, &sh);
    if (extra && (extra->external_bloom || extra->n_jobs)) sh.bloom_file = 0; // compact-many: per-job filters, sized by the caller
    const uint64_t span_total = sh.data_total; // address span of the inputs (sh.data_total becomes the payload bound)
    if (extra && extra->sparse_offsets) sh.data_total = extra->data_bytes;
    (void)span_total;
    if (n_runs > DBEEL_MAX_RUNS) return fail(e, DBEEL_ERR_TOO_MANY_RUNS, "too many runs");
    if (sh.n_total >= 0xFFFFFFFEull) return fail(e, DBEEL_ERR_TOO_MANY_ENTRIES, "too many entries");
    if (out->data_cap < sh.data_total || out->index_cap < sh.n_total * 16 || out->bloom_cap < sh.bloom_file)
        return fail(e, DBEEL_ERR_CAPACITY, "output buffer smaller than dbeel_compact_bound");
    for (uint32_t r = 0; r < n_runs; r++) {
        if ((runs[r].data_len && !runs[r].data) || (runs[r].index_len >= 16 && !runs[r].index))
            return fail(e, DBEEL_ERR_INVALID_ARG, "null run buffer");
        // .data may start anywhere (every access realigns; tables left by dbeel_flush_many / dbeel_compact_many are slices of
        // one output stream); .index is read as 16-byte records
        if ((uintptr_t)runs[r].index & 15) return fail(e, DBEEL_ERR_INVALID_ARG, "device .index buffers must be 16-byte aligned");
    }
    if (((uintptr_t)out->data | (uintptr_t)out->index | (uintptr_t)out->bloom) & 15)
        return fail(e, DBEEL_ERR_INVALID_ARG, "device output buffers must be 16-byte aligned");
    if ((sh.data_total && !out->data) || (sh.n_total && !out->index) || (sh.bloom_file && !out->bloom))
        return fail(e, DBEEL_ERR_INVALID_ARG, "null output buffer");

    dbeel_stats &st = e->stats;
    memset(&st, 0, sizeof st);
    st.input_bytes = sh.data_total + sh.index_total;
    st.entries_in = sh.n_total;
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;

    const uint32_t N = (uint32_t)sh.n_total;
    if (N == 0) return DBEEL_OK; // nothing decodable: empty output, no bloom

    // ---- plan the levels
    Params p;
    memset(&p, 0, sizeof p);
    p.n_runs = n_runs;
    p.n_total = N;
    p.keep_tombstones = o->keep_tombstones ? 1 : 0;
    p.mode_flush = flush ? 1 : 0;
    uint32_t levels = 0;
    const bool many = flush && extra && extra->flush_table;
    const bool jobs = !flush && extra && extra->n_jobs;
    if (jobs) {
        // every job gets the same power-of-two number of leaf slots (its runs, then empty segments): log2(slots)
        // pairwise levels finish every job and never pair runs of two different ones
        uint32_t max_runs = 1;
        for (uint32_t g = 0; g < extra->n_jobs; g++) max_runs = std::max(max_runs, extra->job_first[g + 1] - extra->job_first[g]);
        uint32_t slots = 1;
        while (slots < max_runs) slots <<= 1;
        if ((uint64_t)slots * extra->n_jobs > (1ull << 20)) return fail(e, DBEEL_ERR_TOO_MANY_RUNS, "compact-many: too many run slots");
        p.group_slots = slots;
        p.n_groups = extra->n_jobs;
        p.nseg[0] = slots * extra->n_jobs;
        while ((1u << levels) < slots) {
            p.nseg[levels + 1] = p.nseg[levels] / 2;
            levels++;
        }
    } else if (many) {
        p.n_groups = n_runs;
        // every memtable gets the same power-of-two number of leaf slots (sort tiles), so log2(slots) merge levels
        // finish all memtables and never pair segments of two different ones
        uint64_t max_tiles = 1;
        for (uint32_t r = 0; r < n_runs; r++) {
            const uint64_t t = (runs[r].index_len / DBEEL_INDEX_ENTRY_SIZE + kMergeTile - 1) / kMergeTile;
            max_tiles = t > max_tiles ? t : max_tiles;
        }
        uint32_t slots = 1;
        while (slots < max_tiles) slots <<= 1;
        if (slots > (1u << kMaxLevels) || (uint64_t)slots * n_runs > (1ull << 24))
            return fail(e, DBEEL_ERR_TOO_MANY_ENTRIES, "flush-many: too many sort tiles");
        p.flush_slots = slots;
        p.nseg[0] = slots * n_runs;
        while ((1u << levels) < slots) {
            p.nseg[levels + 1] = p.nseg[levels] / 2;
            levels++;
        }
        for (uint32_t r = 0; r < n_runs; r++)
            if (runs[r].index_len >= DBEEL_INDEX_ENTRY_SIZE) { p.flush_ref_run = r; break; }
    } else {
        p.nseg[0] = flush ? (N + kMergeTile - 1) / kMergeTile : n_runs;
        if (p.nseg[0] > (1u << kMaxLevels)) return fail(e, DBEEL_ERR_TOO_MANY_ENTRIES, "arrival batch too large for one flush");
        while (p.nseg[levels] > 1) {
            p.nseg[levels + 1] = (p.nseg[levels] + 1) / 2;
            levels++;
        }
    }
    p.n_levels = levels;

    // ---- carve the workspace
    uint64_t off = 0;
    // header block (host-initialised, one H2D copy): ctl | runs | first_bad | first_mismatch
    const uint64_t o_ctl = carve_ws(&off, sizeof(Ctl));
    const uint64_t o_runs = carve_ws(&off, sizeof(RunDesc) * n_runs);
    const uint64_t o_fbad = carve_ws(&off, 4ull * n_runs);
    const uint64_t o_fmis = carve_ws(&off, 4ull * n_runs);
    const uint64_t o_groups = carve_ws(&off, jobs ? sizeof(GroupDesc) * (uint64_t)extra->n_jobs : 0);
    const uint64_t header_bytes = off;
    uint64_t o_seg[kMaxLevels + 1], o_tb[kMaxLevels];
    for (uint32_t l = 0; l <= levels; l++) o_seg[l] = carve_ws(&off, sizeof(Seg) * p.nseg[l]);
    for (uint32_t l = 0; l < levels; l++) o_tb[l] = carve_ws(&off, 4ull * (p.nseg[l + 1] + 1));
    const uint64_t tiles_ub = (uint64_t)(N + kFinNominal - 1) / kFinNominal + (p.nseg[0] + 1) / 2; // kFinNominal < kMergeTile: covers both
    const uint64_t bounds_ub = tiles_ub + (p.nseg[0] + 1) / 2 + 1;
    const uint64_t o_part = carve_ws(&off, 4 * bounds_ub);
    const uint64_t o_pext = carve_ws(&off, 4 * bounds_ub);
    const uint64_t o_bnd = carve_ws(&off, 16 * (bounds_ub + 1));
    const uint64_t o_tbnd = carve_ws(&off, 4 * (tiles_ub + 1));
    const uint64_t res_tiles = (uint64_t)(N + kResolveThreads - 1) / kResolveThreads;
    const uint64_t o_tbytes = carve_ws(&off, res_tiles * 8), o_tcount = carve_ws(&off, res_tiles * 4);
    const uint64_t res_chunks = (res_tiles + 1023) / 1024;
    const uint64_t o_cbytes = carve_ws(&off, res_chunks * 8), o_ccount = carve_ws(&off, res_chunks * 4);
    const uint64_t o_reca = carve_ws(&off, 16ull * N), o_recb = carve_ws(&off, 16ull * N);
    const uint64_t o_src = carve_ws(&off, 8ull * N);
    const uint64_t n_groups = p.n_groups;
    const uint64_t o_memtab = carve_ws(&off, n_groups ? 16ull * (n_groups + 1) : 0);
    const uint64_t gather_tiles = (sh.data_total + kGatherTileBytes - 1) / kGatherTileBytes;
    const uint64_t o_tfirst = carve_ws(&off, 4ull * (gather_tiles + 2));
    const bool ref_reader = !flush && !jobs && (o->flags & DBEEL_FLAG_REFERENCE_READER);
    const uint64_t o_fix = carve_ws(&off, ref_reader ? 16ull * N : 0);
    // single compaction: the last merge level, resolve, the offsets scan and the .index writes in one persistent kernel
    const bool fused_final = e->fused_final && e->fin_ctas_per_sm > 0 && !flush && !jobs && !many && levels >= 1;
    const uint64_t fin_tiles_ub = (uint64_t)(N + kFinNominal - 1) / kFinNominal + 1;
    p.fin_tile = fused_final ? (uint32_t)kFinNominal : 0u;
    const uint64_t scan_bytes = fused_final ? 16ull * fin_tiles_ub + 64 : 0;
    const uint64_t o_scan = carve_ws(&off, scan_bytes);
    int rc = ensure_device(e, &e->ws, &e->ws_cap, off);
    if (rc) return rc;
    rc = ensure_pinned(e, header_bytes + align_up(sizeof(Ctl), 64) + 64 + (n_groups ? 16ull * (n_groups + 1) : 0));
    if (rc) return rc;

    uint8_t *ws = e->ws;
    p.ctl = reinterpret_cast<Ctl *>(ws + o_ctl);
    p.runs = reinterpret_cast<RunDesc *>(ws + o_runs);
    p.first_bad = reinterpret_cast<uint32_t *>(ws + o_fbad);
    p.first_mismatch = reinterpret_cast<uint32_t *>(ws + o_fmis);
    for (uint32_t l = 0; l <= levels; l++) p.seg[l] = reinterpret_cast<Seg *>(ws + o_seg[l]);
    for (uint32_t l = 0; l < levels; l++) p.tile_base[l] = reinterpret_cast<uint32_t *>(ws + o_tb[l]);
    p.part = reinterpret_cast<uint32_t *>(ws + o_part);
    p.part_ext = reinterpret_cast<uint32_t *>(ws + o_pext);
    p.bnd = reinterpret_cast<uint4 *>(ws + o_bnd);
    p.tile_bnd = reinterpret_cast<uint32_t *>(ws + o_tbnd);
    p.tile_bytes = reinterpret_cast<unsigned long long *>(ws + o_tbytes);
    p.tile_count = reinterpret_cast<uint32_t *>(ws + o_tcount);
    p.chunk_bytes = reinterpret_cast<unsigned long long *>(ws + o_cbytes);
    p.chunk_count = reinterpret_cast<uint32_t *>(ws + o_ccount);
    p.rec_a = reinterpret_cast<Rec *>(ws + o_reca);
    p.rec_b = reinterpret_cast<Rec *>(ws + o_recb);
    p.src_ptr = reinterpret_cast<unsigned long long *>(ws + o_src);
    p.tile_first = reinterpret_cast<uint32_t *>(ws + o_tfirst);
    p.tile_first_n = (uint32_t)(gather_tiles + 2);
    p.data_bound = sh.data_total;
    p.mem_table = reinterpret_cast<unsigned long long *>(ws + o_memtab);
    p.ref_reader = ref_reader ? 1 : 0;
    p.fix_index = reinterpret_cast<uint4 *>(ws + o_fix);
    p.scan_state = reinterpret_cast<unsigned long long *>(ws + o_scan);
    p.out_data = static_cast<uint8_t *>(out->data);
    p.out_index = static_cast<uint4 *>(out->index);

    // ---- header block
    uint8_t *h = e->pin;
    memset(h, 0, header_bytes);
    RunDesc *hr = reinterpret_cast<RunDesc *>(h + o_runs);
    uint32_t *hb = reinterpret_cast<uint32_t *>(h + o_fbad), *hm = reinterpret_cast<uint32_t *>(h + o_fmis);
    uint32_t base = 0;
    for (uint32_t r = 0; r < n_runs; r++) {
        hr[r].data = static_cast<const uint8_t *>(runs[r].data);
        hr[r].off_base = extra && extra->off_base ? extra->off_base[r] : 0;
        hr[r].data_len = hr[r].off_base + runs[r].data_len;
        hr[r].index = static_cast<const uint4 *>(runs[r].index);
        hr[r].n_in = (uint32_t)(runs[r].index_len / DBEEL_INDEX_ENTRY_SIZE);
        hr[r].base = base;
        hb[r] = hr[r].n_in;
        hm[r] = 0xFFFFFFFFu;
        base += hr[r].n_in;
    }
    if (jobs) {
        GroupDesc *hg = reinterpret_cast<GroupDesc *>(h + o_groups);
        for (uint32_t g = 0; g < extra->n_jobs; g++) {
            const uint32_t r0 = extra->job_first[g], r1 = extra->job_first[g + 1];
            hg[g].first_run = r0;
            hg[g].n_runs = r1 - r0;
            hg[g].pos_end = r1 > r0 ? hr[r1 - 1].base + hr[r1 - 1].n_in : (r0 < n_runs ? hr[r0].base : base);
            hg[g].keep_tombstones = extra->job_keep[g] ? 1 : 0;
            hg[g].bloom = extra->job_bloom[g];
        }
        p.groups = reinterpret_cast<const GroupDesc *>(ws + o_groups);
    }

    // ---- bloom
    uint8_t seed[32];
    if (sh.bloom_file) {
        if (o->bloom_seed) {
            memcpy(seed, o->bloom_seed, 32);
        } else { // Bloom::new -> getrandom(&mut seed)
            FILE *f = fopen("/dev/urandom", "rb");
            if (!f || fread(seed, 1, 32, f) != 32) {
                if (f) fclose(f);
                return fail(e, DBEEL_ERR_INVALID_ARG, "no entropy source for the bloom seed");
            }
            fclose(f);
        }
        p.bloom.words = reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(out->bloom) + 8);
        p.bloom.bits = sh.bloom_bits;
        p.bloom.bits_magic = (uint64_t)((((unsigned __int128)1) << 64) / sh.bloom_bits);
        p.bloom.k_num = sh.bloom_k;
        for (int i = 0; i < 4; i++) memcpy(&p.bloom.sip[i], seed + 8 * i, 8);
    }
    if (extra) {
        p.sparse_offsets = extra->sparse_offsets ? 1 : 0;
        p.out_offset_base = extra->out_offset_base;
        if (extra->external_bloom) p.bloom = extra->bloom;
    }

    cudaStream_t s = e->stream;
    uint32_t launches = 0;
    // The header goes down and the control block comes back through kernels that touch the mapped pinned block, not
    // through cudaMemcpyAsync: a small copy on this stream would queue on a copy engine behind whatever bulk transfer
    // of the pipelined host path is in flight there (measured: every partition's kernels waited for the previous
    // partition's 200 MB D2H).  The compute stream carries kernels and event records only.
    CU(cudaEventRecord(e->ev[EV_START], s)); // ms_total covers the header upload and the filter's memset too
    launch_k(e, k_copy_words, (uint32_t)((header_bytes / 4 + 255) / 256), 256, 0, s, reinterpret_cast<uint32_t *>(ws),
             reinterpret_cast<const uint32_t *>(e->pin_dev), (uint32_t)(header_bytes / 4));
    launches++;
    if (sh.bloom_file) CU(cudaMemsetAsync(out->bloom, 0, sh.bloom_file, s));
    if (scan_bytes) CU(cudaMemsetAsync(ws + o_scan, 0, scan_bytes, s));

    // ---- K0/K1: prefix, validate, extract (+ conditional redo when a run was truncated)
    const uint32_t g256 = (N + 255) / 256;
    const uint32_t gext = (N + 256 * kExtractEPT - 1) / (256 * kExtractEPT);
    auto launch_extract = [&](uint32_t grid, int mode) {
        if (ref_reader) launch_k(e, k_extract<true, true>, grid, 256, 0, s, p, mode);
        else if (e->narrow_loads && e->extract_persist > 0 && mode == 0) // one resident wave, index records fetched a step ahead
            launch_k(e, k_extract<true, false, true>, std::min<uint32_t>(grid, (uint32_t)(e->sm_count * e->extract_persist)), 256, 0, s, p, mode);
        else if (e->narrow_loads) launch_k(e, k_extract<true, false>, grid, 256, 0, s, p, mode);
        else launch_k(e, k_extract<false, false>, grid, 256, 0, s, p, mode);
    };
    if (flush) {
        launch_k(e, k_flush_prefix_init, 1, 1, 0, s, p);
        launch_k(e, k_flush_prefix, g256, 256, 0, s, p);
        launch_extract(gext, 0);
        launch_k(e, k_plan, 1, 1024, 0, s, p);
        launch_k(e, k_block_sort, p.nseg[0], kMergeThreads, 0, s, p);
    } else {
        launch_k(e, k_common_prefix, 1, 32, 0, s, p, 0);
        launch_extract(gext, 0);
        if (ref_reader) { // all four are no-ops unless an index record disagrees with its .data (lsm_tree.rs:1158-1170)
            launch_k(e, k_ref_repair, n_runs, 1024, 0, s, p);
            launch_k(e, k_ref_reset, 1, 256, 0, s, p);
            launch_k(e, k_common_prefix, 1, 32, 0, s, p, 2);
            launch_extract(gext < 592 ? gext : 592, 2);
            launches += 4;
        }
        launch_k(e, k_common_prefix, 1, 32, 0, s, p, 1); // both no-ops unless a run was truncated
        launch_extract(gext < 592 ? gext : 592, 1);
        launch_k(e, k_plan, 1, 1024, 0, s, p);
    }
    launches += 5;
    if (!flush && (o->flags & DBEEL_FLAG_VERIFY_SORTED)) {
        launch_k(e, k_verify_sorted, g256, 256, 0, s, p);
        launches++;
    }
    const bool stage_ev = e->stage_events != 0;
    if (stage_ev) CU(cudaEventRecord(e->ev[EV_EXTRACT], s));

    // ---- K2/K3: merge levels, ping-pong between rec_a and rec_b
    const Rec *src = p.rec_a;
    Rec *dst = p.rec_b;
    if (sh.bloom_file) { // independent of everything else: its launch overlaps the merges
        launch_k(e, k_bloom_frame, 1, 1, 0, s, static_cast<uint8_t *>(out->bloom), sh.bloom_words, p.bloom);
        launches++;
    }
    for (uint32_t l = 0; l < levels; l++) {
        uint32_t pairs = p.nseg[l + 1];
        const bool last_fused = fused_final && l + 1 == levels;
        const uint64_t tl = last_fused ? kFinNominal : kMergeTile;
        uint64_t t_ub = (uint64_t)(N + tl - 1) / tl + pairs;
        uint64_t b_ub = t_ub + pairs;
        if (last_fused && stage_ev) CU(cudaEventRecord(e->ev[EV_MERGE], s)); // the fused last level is booked under ms_resolve
        launch_k(e, k_merge_partition, (uint32_t)((b_ub + 7) / 8), kPartitionThreads, 0, s, p, l, src); // one warp per boundary
        if (last_fused) { // persistent; merged tile -> resolve -> chained scan -> .index, all from shared memory
            uint64_t grid = (uint64_t)e->sm_count * e->fin_ctas_per_sm;
            if (grid > t_ub) grid = t_ub;
            if (e->narrow_loads) launch_k(e, k_merge_final<true>, (uint32_t)grid, kFinThreads, kFinSmem, s, p, l, src);
            else launch_k(e, k_merge_final<false>, (uint32_t)grid, kFinThreads, kFinSmem, s, p, l, src);
        } else { // persistent, TMA bulk loads / stores + mbarrier
            uint64_t grid = (uint64_t)e->sm_count * kMergeCtasPerSM;
            if (grid > t_ub) grid = t_ub;
            launch_k(e, k_merge_tma, (uint32_t)grid, kMergeThreads, 2 * kMergeBufRecs * sizeof(Rec), s, p, l, src, dst);
        }
        launches += 2;
        if (last_fused) break; // src stays the last level's input: nothing was written to dst
        const Rec *t = src;
        src = dst;
        dst = const_cast<Rec *>(t);
    }
    if (!fused_final && stage_ev) CU(cudaEventRecord(e->ev[EV_MERGE], s));

    // ---- K4: resolve + scan + .index
    if (jobs) {
        launch_k(e, k_bloom_frames, (extra->n_jobs + 127) / 128, 128, 0, s, p.groups, extra->n_jobs);
        launches++;
    }
    uint4 *res = reinterpret_cast<uint4 *>(dst); // the ping-pong buffer that does not hold the merged order
    if (!fused_final) {
        if (e->narrow_loads) launch_k(e, k_resolve<true>, (uint32_t)res_tiles, kResolveThreads, 0, s, p, src, res);
        else launch_k(e, k_resolve<false>, (uint32_t)res_tiles, kResolveThreads, 0, s, p, src, res);
        launch_k(e, k_scan_tiles, (uint32_t)res_chunks, 1024, 0, s, p);
        launch_k(e, k_scan_chunks, 1, 1024, 0, s, p);
        launch_k(e, k_emit, (uint32_t)res_tiles, kResolveThreads, 0, s, p, res);
        launches += 4;
    }
    if (n_groups) {
        launch_k(e, k_flush_table, (uint32_t)((n_groups + 1 + 127) / 128), 128, 0, s, p, res);
        launches++;
    }
    if (stage_ev) CU(cudaEventRecord(e->ev[EV_RESOLVE], s));

    // ---- K5: gather + bloom (fused epilogue)
    if (gather_tiles) launch_k(e, k_gather_h, (uint32_t)gather_tiles, kGhThreads, 0, s, p);
    launches++;
    if (jobs) { // per-job filters: their own pass over the output entries
        launch_k(e, k_bloom_many, g256, 256, 0, s, p);
        launches++;
    }
    if (n_groups) { // only now may the .index offsets become file-relative: the gather kernel reads them as stream offsets
        launch_k(e, k_rebase_index, g256, 256, 0, s, p);
        launches++;
    }
    CU(cudaEventRecord(e->ev[EV_GATHER], s));
    CU(cudaGetLastError());

    // ---- control block back
    static_assert(sizeof(Ctl) % 4 == 0, "the control block is published word by word");
    Ctl *hc = reinterpret_cast<Ctl *>(e->pin + header_bytes);
    const uint64_t o_hmt = header_bytes + align_up(sizeof(Ctl), 64);
    unsigned long long *hmt = reinterpret_cast<unsigned long long *>(e->pin + o_hmt);
    launch_k(e, k_publish, 1, 256, 0, s, reinterpret_cast<uint32_t *>(e->pin_dev + header_bytes), reinterpret_cast<const uint32_t *>(p.ctl),
             (uint32_t)(sizeof(Ctl) / 4), reinterpret_cast<uint32_t *>(e->pin_dev + o_hmt),
             reinterpret_cast<const uint32_t *>(p.mem_table), n_groups ? (uint32_t)(4 * (n_groups + 1)) : 0u);
    launches++;
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));

    st.kernel_launches = launches;
    st.merge_passes = levels;
    st.key_prefix_len = hc->prefix_len;
    st.entries_valid = hc->total;
    st.runs_truncated = hc->runs_truncated;
    st.index_repaired = (hc->flags & kFlagRepaired) ? 1 : 0;
    cudaEventElapsedTime(&st.ms_total, e->ev[EV_START], e->ev[EV_GATHER]);
    if (stage_ev) {
        cudaEventElapsedTime(&st.ms_extract, e->ev[EV_START], e->ev[EV_EXTRACT]);
        cudaEventElapsedTime(&st.ms_merge, e->ev[EV_EXTRACT], e->ev[EV_MERGE]);
        cudaEventElapsedTime(&st.ms_resolve, e->ev[EV_MERGE], e->ev[EV_RESOLVE]);
        cudaEventElapsedTime(&st.ms_gather, e->ev[EV_RESOLVE], e->ev[EV_GATHER]);
    }
    if (hc->flags & (kFlagUnsorted | kFlagVerifyFailed))
        return fail(e, DBEEL_ERR_UNSORTED_RUN, "an input run is not strictly ascending by key");
    if (hc->out_data_len > sh.data_total) // only possible with a caller-supplied payload bound (sparse batches)
        return fail(e, DBEEL_ERR_CAPACITY, "payload bound of a sparse batch is lower than the bytes it holds");

    out->data_len = hc->out_data_len;
    out->items_written = hc->out_items;
    out->index_len = (uint64_t)hc->out_items * 16;
    out->bloom_len = sh.bloom_file;
    st.entries_out = hc->out_items;
    st.output_bytes = out->data_len + out->index_len + out->bloom_len;
    st.gather_bytes = 2 * out->data_len + out->index_len + 8ull * hc->out_items; // read + write payload, read index + src_ptr
    st.partitions = 1;
    if (jobs) {
        for (uint32_t g = 0; g < extra->n_jobs; g++) {
            dbeel_job_result &row = extra->job_results[g];
            row.data_off = hmt[2 * g];
            row.data_len = hmt[2 * (g + 1)] - hmt[2 * g];
            row.items_written = hmt[2 * (g + 1) + 1] - hmt[2 * g + 1];
            row.index_off = hmt[2 * g + 1] * 16;
            row.index_len = row.items_written * 16;
        }
    }
    if (many) {
        for (uint32_t r = 0; r < n_runs; r++) {
            dbeel_flush_table &row = extra->flush_table[r];
            row.data_off = hmt[2 * r];
            row.data_len = hmt[2 * (r + 1)] - hmt[2 * r];
            row.items = hmt[2 * (r + 1) + 1] - hmt[2 * r + 1];
            row.index_off = hmt[2 * r + 1] * 16;
            row.index_len = row.items * 16;
        }
    }
    return DBEEL_OK;
}

// ------------------------------------------------------------------------------------
// Pipelined host entry point.  A compaction whose inputs live in host memory is PCIe-bound
// (transfers take several times as long as the kernels), so the job is cut into key-range
// partitions: partition i's slices of every run go down on one stream while partition i-1 is
// merged and partition i-2's output goes up on a third -- both PCIe directions stay busy.
// Every key lives in exactly one partition (all runs are cut at the same splitter keys with
// lower_bound), partitions are emitted in key order, .index offsets continue across partitions
// (out_offset_base) and all partitions set bits in one shared bloom filter sized for the whole
// compaction, so the output files are byte-identical to the single-shot path.

constexpr int kFallbackSingleShot = -1000; // internal: inputs need the single-shot path (corrupt / odd)

struct HostRun {
    const uint8_t *data;
    uint64_t data_len;
    const uint8_t *index;
    uint64_t n;
};

struct HostRec {
    uint64_t off;
    uint32_t ks, fs;
};

inline bool host_rec(const HostRun &r, uint64_t i, HostRec *out) {
    const uint8_t *p = r.index + 16 * i;
    memcpy(&out->off, p, 8);
    memcpy(&out->ks, p + 8, 4);
    memcpy(&out->fs, p + 12, 4);
    return out->ks >= 8 && (uint64_t)out->fs >= (uint64_t)out->ks + 24 && out->off <= r.data_len &&
           (uint64_t)out->fs <= r.data_len - out->off;
}

inline int host_key_cmp(const uint8_t *a, uint32_t al, const uint8_t *b, uint32_t bl) {
    const uint32_t m = al < bl ? al : bl;
    const int c = m ? memcmp(a, b, m) : 0;
    if (c) return c;
    return (al > bl) - (al < bl);
}

struct Splitter {
    const uint8_t *key;
    uint32_t klen;
    uint64_t weight;
};

// io != null: the streaming variant (dbeel_compact_stream).  The runs' pointers are ignored: the .index files are pulled
// whole into pinned memory first (16 bytes per entry), the keys the planner looks at come through small reads, and the
// .data slices of partition c travel file -> pinned ring -> device while the outputs travel device -> pinned ring -> file
// on the threads of a StreamPump (host/stream_pump.h).
int run_job_host_pipelined(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *o,
                           dbeel_out *out, const JobShape &sh, const dbeel_stream_io *io = nullptr) {
    // ---- 1. splitters from weighted samples of every run
    std::vector<HostRun> hr(n_runs);
    for (uint32_t r = 0; r < n_runs; r++)
        hr[r] = HostRun{io ? nullptr : static_cast<const uint8_t *>(runs[r].data), runs[r].data_len,
                        io ? nullptr : static_cast<const uint8_t *>(runs[r].index), runs[r].index_len / DBEEL_INDEX_ENTRY_SIZE};
    uint64_t P = (sh.data_total + sh.index_total + e->partition_bytes - 1) / e->partition_bytes;
    if (P > 64) P = 64;
    if (P < 2) return kFallbackSingleShot;
    if (io) { // the .index files, whole, into page-locked memory (they are also what the H2D copies of the index slices read)
        std::vector<uint64_t> ioff(n_runs);
        uint64_t need = 0;
        for (uint32_t r = 0; r < n_runs; r++) {
            ioff[r] = need;
            need += align_up(hr[r].n * 16 + 16, kAlign);
        }
        int rc = ensure_host(e, &e->pin_index, &e->pin_index_cap, need);
        if (rc) return rc;
        std::vector<StreamPump::ReadTask> rt;
        for (uint32_t r = 0; r < n_runs; r++) {
            hr[r].index = e->pin_index + ioff[r];
            for (uint64_t done = 0; done < hr[r].n * 16; done += StreamPump::kPiece)
                rt.push_back(StreamPump::ReadTask{0, r, DBEEL_STREAM_INDEX, done, std::min<uint64_t>(StreamPump::kPiece, hr[r].n * 16 - done),
                                                  e->pin_index + ioff[r] + done});
        }
        rc = parallel_pieces(rt.size(), [&](size_t k) { return io->read(io->ctx, rt[k].run, rt[k].kind, rt[k].off, rt[k].len, rt[k].dst); });
        if (rc) return fail(e, rc, "stream read callback failed (.index)");
    }
    // a key the planner compares: in memory, or fetched through the read callback into `store`
    std::deque<std::vector<uint8_t>> key_store;
    int key_rc = 0;
    auto key_of = [&](uint32_t r, const HostRec &rec, bool keep) -> const uint8_t * {
        if (!io) return hr[r].data + rec.off + 8;
        if (!keep && !key_store.empty()) key_store.pop_back(); // the previous probe's scratch
        key_store.emplace_back(rec.ks - 8 ? rec.ks - 8 : 1);
        if (rec.ks > 8) {
            const int rc = io->read(io->ctx, r, DBEEL_STREAM_DATA, rec.off + 8, rec.ks - 8, key_store.back().data());
            if (rc && !key_rc) key_rc = rc;
        }
        return key_store.back().data();
    };
    constexpr uint64_t kSamples = 256;
    std::vector<Splitter> samples;
    for (uint32_t r = 0; r < n_runs; r++) {
        const uint64_t n = hr[r].n;
        if (!n) continue;
        const uint64_t cnt = n < kSamples ? n : kSamples;
        for (uint64_t q = 0; q < cnt; q++) {
            const uint64_t i = (2 * q + 1) * n / (2 * cnt);
            HostRec rec;
            if (!host_rec(hr[r], i, &rec)) return kFallbackSingleShot;
            samples.push_back(Splitter{key_of(r, rec, true), rec.ks - 8, n / cnt + 1});
        }
    }
    if (key_rc) return fail(e, key_rc, "stream read callback failed (sample keys)");
    if (io) key_store.emplace_back(1); // scratch slot the probes below recycle
    if (samples.empty()) return kFallbackSingleShot;
    std::sort(samples.begin(), samples.end(), [](const Splitter &a, const Splitter &b) {
        return host_key_cmp(a.key, a.klen, b.key, b.klen) < 0;
    });
    uint64_t wsum = 0;
    for (auto &sm : samples) wsum += sm.weight;
    // Partition sizes: the pipeline's fill (nothing to merge until the first partition is down) and drain (nothing but
    // the last partition's D2H) cost one partition's transfer each, so the first and last partitions are small:
    // 1/4, 1/2, 1, 1, ..., 1, 1/2, 1/4 of the nominal size.
    std::vector<double> share;
    if (P >= 4 && e->partition_taper) {
        share = {0.25, 0.5};
        const uint64_t mid = P - 1 > 59 ? 59 : P - 1; // 2P-1 quarter units short of the total: one more full partition
        for (uint64_t k = 0; k < mid; k++) share.push_back(1.0);
        share.push_back(0.5);
        share.push_back(0.25);
    } else {
        share.assign(P, 1.0);
    }
    double share_sum = 0;
    for (double v : share) share_sum += v;
    std::vector<Splitter> cuts;
    {
        uint64_t acc = 0;
        size_t next = 0; // the cut after partition `next`
        double target = share[0] / share_sum;
        for (auto &sm : samples) {
            acc += sm.weight;
            if (next + 1 < share.size() && (double)acc >= target * (double)wsum) {
                if (cuts.empty() || host_key_cmp(cuts.back().key, cuts.back().klen, sm.key, sm.klen) < 0) cuts.push_back(sm);
                while (next + 1 < share.size() && (double)acc >= target * (double)wsum) {
                    next++;
                    target += share[next] / share_sum;
                }
            }
        }
    }
    const uint32_t np = (uint32_t)cuts.size() + 1;
    if (np < 2) return kFallbackSingleShot;

    // ---- 2. cut every run at every splitter (lower_bound: equal keys of all runs land in the same partition)
    std::vector<std::vector<uint64_t>> lo(n_runs, std::vector<uint64_t>(np + 1, 0));
    std::vector<std::vector<uint64_t>> boff(n_runs, std::vector<uint64_t>(np + 1, 0)); // .data offset at each cut
    for (uint32_t r = 0; r < n_runs; r++) {
        const uint64_t n = hr[r].n;
        lo[r][np] = n;
        for (uint32_t c = 0; c < np - 1; c++) {
            uint64_t a = c ? lo[r][c] : 0, b = n;
            while (a < b) {
                const uint64_t mid = (a + b) >> 1;
                HostRec rec;
                if (!host_rec(hr[r], mid, &rec)) return kFallbackSingleShot;
                if (host_key_cmp(key_of(r, rec, false), rec.ks - 8, cuts[c].key, cuts[c].klen) < 0) a = mid + 1; else b = mid;
            }
            lo[r][c + 1] = a;
        }
        uint64_t end = 0;
        if (n) {
            HostRec last;
            if (!host_rec(hr[r], n - 1, &last)) return kFallbackSingleShot;
            end = last.off + last.fs;
        }
        for (uint32_t c = 0; c <= np; c++) {
            const uint64_t i = lo[r][c];
            if (i >= n) { boff[r][c] = end; continue; }
            HostRec rec;
            if (!host_rec(hr[r], i, &rec)) return kFallbackSingleShot;
            if (i) { // the offsets chain must hold across the cut (inside a slice the GPU checks it)
                HostRec prev;
                if (!host_rec(hr[r], i - 1, &prev) || prev.off + prev.fs != rec.off) return kFallbackSingleShot;
            } else if (rec.off != 0) {
                return kFallbackSingleShot;
            }
            boff[r][c] = rec.off;
        }
    }

    if (key_rc) return fail(e, key_rc, "stream read callback failed (splitter probes)");

    // ---- 3. staging: two input and two output buffers sized for the largest partition
    uint64_t max_in = 0, max_out = 0;
    for (uint32_t c = 0; c < np; c++) {
        uint64_t in = 0, d = 0, ix = 0;
        for (uint32_t r = 0; r < n_runs; r++) {
            const uint64_t dl = boff[r][c + 1] - boff[r][c], il = (lo[r][c + 1] - lo[r][c]) * 16;
            in += align_up(dl + 32, kAlign) + align_up(il + 16, kAlign);
            d += dl;
            ix += il;
        }
        const uint64_t o2 = align_up(d + 16, kAlign) + align_up(ix + 16, kAlign);
        max_in = in > max_in ? in : max_in;
        max_out = o2 > max_out ? o2 : max_out;
    }
    int rc = ensure_device(e, &e->stage_in, &e->stage_in_cap, max_in);
    if (!rc) rc = ensure_device(e, &e->stage_in2, &e->stage_in2_cap, max_in);
    if (!rc) rc = ensure_device(e, &e->stage_out, &e->stage_out_cap, max_out);
    if (!rc) rc = ensure_device(e, &e->stage_out2, &e->stage_out2_cap, max_out);
    if (!rc && sh.bloom_file) rc = ensure_device(e, &e->bloom_dev, &e->bloom_dev_cap, sh.bloom_file + 16);
    if (!rc) rc = ensure_copy_streams(e);
    if (rc) return rc;
    uint8_t *sin[2] = {e->stage_in, e->stage_in2}, *sout[2] = {e->stage_out, e->stage_out2};
    // streaming: R-slot pinned rings on both sides, one event per partition for the writer threads, the pump itself.
    // Declared in this order so that the pump's threads are joined before the events they wait on are destroyed.
    struct EventList {
        std::vector<cudaEvent_t> ev;
        ~EventList() { for (auto &x : ev) if (x) cudaEventDestroy(x); }
    } ev_out;
    std::unique_ptr<StreamPump> pump;
    const uint32_t R = (uint32_t)std::max(2, e->stream_ring);
    if (io) {
        rc = ensure_host(e, &e->ring_in, &e->ring_in_cap, (uint64_t)R * max_in);
        if (!rc) rc = ensure_host(e, &e->ring_out, &e->ring_out_cap, (uint64_t)R * max_out);
        if (!rc && sh.bloom_file) rc = ensure_host(e, &e->pin_bloom, &e->pin_bloom_cap, sh.bloom_file);
        if (rc) return rc;
        ev_out.ev.assign(np, nullptr);
        for (uint32_t c = 0; c < np; c++) CU(cudaEventCreateWithFlags(&ev_out.ev[c], cudaEventDisableTiming | cudaEventBlockingSync));
        const int dev = e->device;
        EventList *evl = &ev_out;
        pump.reset(new StreamPump(io, np, R, stream_threads(), [evl](uint32_t c) { cudaEventSynchronize(evl->ev[c]); }, [dev]() { cudaSetDevice(dev); }));
        for (uint32_t c = 0; c < np; c++) {
            uint8_t *slot = e->ring_in + (uint64_t)(c % R) * max_in;
            uint64_t pos = 0;
            for (uint32_t r = 0; r < n_runs; r++) {
                const uint64_t dl = boff[r][c + 1] - boff[r][c], il = (lo[r][c + 1] - lo[r][c]) * 16;
                if (dl) pump->add_read(c, r, DBEEL_STREAM_DATA, boff[r][c], dl, slot + pos);
                pos += align_up(dl + 32, kAlign) + align_up(il + 16, kAlign);
            }
        }
        pump->start();
    }

    // ---- 4. the shared bloom filter
    JobExtra ex;
    ex.external_bloom = true;
    if (sh.bloom_file) {
        uint8_t seed[32];
        if (o->bloom_seed) {
            memcpy(seed, o->bloom_seed, 32);
        } else {
            FILE *f = fopen("/dev/urandom", "rb");
            if (!f || fread(seed, 1, 32, f) != 32) {
                if (f) fclose(f);
                return fail(e, DBEEL_ERR_INVALID_ARG, "no entropy source for the bloom seed");
            }
            fclose(f);
        }
        ex.bloom.words = reinterpret_cast<uint32_t *>(e->bloom_dev + 8);
        ex.bloom.bits = sh.bloom_bits;
        ex.bloom.bits_magic = (uint64_t)((((unsigned __int128)1) << 64) / sh.bloom_bits);
        ex.bloom.k_num = sh.bloom_k;
        for (int i = 0; i < 4; i++) memcpy(&ex.bloom.sip[i], seed + 8 * i, 8);
        CU(cudaMemsetAsync(e->bloom_dev, 0, sh.bloom_file, e->stream));
        k_bloom_frame<<<1, 1, 0, e->stream>>>(e->bloom_dev, sh.bloom_words, ex.bloom);
    }

    // ---- 5. the pipeline
    const bool trace = getenv("DBEEL_TRACE") != nullptr; // per-partition timeline on stderr (debug aid)
    std::vector<cudaEvent_t> tev;
    if (trace) {
        tev.resize(6 * (size_t)np);
        for (auto &ev : tev) CU(cudaEventCreate(&ev));
    }
    std::vector<uint64_t> off_base(n_runs);
    std::vector<dbeel_run> dr(n_runs);
    auto enqueue_h2d = [&](uint32_t c) -> int {
        uint8_t *base = sin[c & 1];
        uint64_t pos = 0;
        const uint8_t *slot = io ? e->ring_in + (uint64_t)(c % R) * max_in : nullptr;
        if (io) { // partition c's slices have to be in their ring slot
            const int prc = pump->wait_reads(c);
            if (prc) return fail(e, prc, "stream read callback failed (.data)");
        }
        if (trace) CU(cudaEventRecord(tev[6 * c + 0], e->s_h2d));
        for (uint32_t r = 0; r < n_runs; r++) {
            const uint64_t dl = boff[r][c + 1] - boff[r][c], il = (lo[r][c + 1] - lo[r][c]) * 16;
            if (dl) CU(cudaMemcpyAsync(base + pos, io ? slot + pos : hr[r].data + boff[r][c], dl, cudaMemcpyHostToDevice, e->s_h2d));
            pos += align_up(dl + 32, kAlign);
            if (il) CU(cudaMemcpyAsync(base + pos, hr[r].index + 16 * lo[r][c], il, cudaMemcpyHostToDevice, e->s_h2d));
            pos += align_up(il + 16, kAlign);
        }
        CU(cudaEventRecord(e->ev_h2d[c & 1], e->s_h2d));
        if (trace) CU(cudaEventRecord(tev[6 * c + 1], e->s_h2d));
        return DBEEL_OK;
    };
    dbeel_stats total = {};
    total.input_bytes = sh.data_total + sh.index_total;
    total.entries_in = sh.n_total;
    uint64_t out_data = 0, out_items = 0;
    uint8_t *h_data = static_cast<uint8_t *>(out->data), *h_index = static_cast<uint8_t *>(out->index);
    CU(cudaEventRecord(e->ev[EV_H2D0], e->stream));
    rc = enqueue_h2d(0);
    if (!rc && np > 1) rc = enqueue_h2d(1);
    if (rc) return rc;
    bool truncated = false;
    for (uint32_t c = 0; c < np; c++) {
        uint8_t *base = sin[c & 1];
        uint64_t pos = 0, dsum = 0, isum = 0;
        for (uint32_t r = 0; r < n_runs; r++) {
            const uint64_t dl = boff[r][c + 1] - boff[r][c], il = (lo[r][c + 1] - lo[r][c]) * 16;
            off_base[r] = boff[r][c];
            dr[r].data = base + pos - boff[r][c]; // biased: .data offset `off` lives at data + off
            dr[r].data_len = dl;
            pos += align_up(dl + 32, kAlign);
            dr[r].index = base + pos;
            dr[r].index_len = il;
            pos += align_up(il + 16, kAlign);
            dsum += dl;
            isum += il;
        }
        dbeel_out dout = {};
        dout.data = sout[c & 1];
        dout.data_cap = dsum;
        dout.index = sout[c & 1] + align_up(dsum + 16, kAlign);
        dout.index_cap = isum;
        ex.off_base = off_base.data();
        ex.out_offset_base = out_data;
        CU(cudaStreamWaitEvent(e->stream, e->ev_h2d[c & 1], 0));
        if (c >= 2) CU(cudaStreamWaitEvent(e->stream, e->ev_d2h[c & 1], 0)); // output buffer c&1 drained
        if (trace) CU(cudaEventRecord(tev[6 * c + 2], e->stream));
        rc = run_job_device(e, dr.data(), n_runs, o, false, &dout, &ex); // syncs e->stream
        if (rc) break;
        if (io) pump->release_input(c); // the kernels have read device buffer c & 1, which the H2D out of ring slot c mod R filled
        const dbeel_stats &ps = e->stats;
        if (ps.runs_truncated || ps.index_repaired) { truncated = true; break; } // the slices were cut by index offsets: redo exactly
        total.entries_valid += ps.entries_valid;
        total.kernel_launches += ps.kernel_launches;
        total.merge_passes = ps.merge_passes > total.merge_passes ? ps.merge_passes : total.merge_passes;
        total.key_prefix_len = ps.key_prefix_len;
        total.ms_total += ps.ms_total;
        total.ms_extract += ps.ms_extract;
        total.ms_merge += ps.ms_merge;
        total.ms_resolve += ps.ms_resolve;
        total.ms_gather += ps.ms_gather;
        total.gather_bytes += ps.gather_bytes;
        CU(cudaEventRecord(e->ev_comp[c & 1], e->stream));
        if (trace) CU(cudaEventRecord(tev[6 * c + 3], e->stream));
        CU(cudaStreamWaitEvent(e->s_d2h, e->ev_comp[c & 1], 0));
        if (trace) CU(cudaEventRecord(tev[6 * c + 4], e->s_d2h));
        if (io) { // device -> ring slot c mod R (once partition c - R has left it) -> the writer threads
            rc = pump->wait_out_slot(c);
            if (rc) { fail(e, rc, "stream write callback failed"); break; }
            uint8_t *oslot = e->ring_out + (uint64_t)(c % R) * max_out;
            uint8_t *oindex = oslot + align_up(dout.data_len + 16, kAlign);
            if (dout.data_len) CU(cudaMemcpyAsync(oslot, dout.data, dout.data_len, cudaMemcpyDeviceToHost, e->s_d2h));
            if (dout.index_len) CU(cudaMemcpyAsync(oindex, dout.index, dout.index_len, cudaMemcpyDeviceToHost, e->s_d2h));
            CU(cudaEventRecord(ev_out.ev[c], e->s_d2h));
            StreamPump::OutPart op;
            op.data = oslot; op.data_len = dout.data_len; op.data_off = out_data;
            op.index = oindex; op.index_len = dout.index_len; op.index_off = 16 * out_items;
            pump->publish_out(c, op);
        } else {
            if (dout.data_len) CU(cudaMemcpyAsync(h_data + out_data, dout.data, dout.data_len, cudaMemcpyDeviceToHost, e->s_d2h));
            if (dout.index_len) CU(cudaMemcpyAsync(h_index + 16 * out_items, dout.index, dout.index_len, cudaMemcpyDeviceToHost, e->s_d2h));
        }
        CU(cudaEventRecord(e->ev_d2h[c & 1], e->s_d2h));
        if (trace) CU(cudaEventRecord(tev[6 * c + 5], e->s_d2h));
        out_data += dout.data_len;
        out_items += dout.items_written;
        if (c + 2 < np) { // input buffer c&1 is free again (the job that read it has completed)
            rc = enqueue_h2d(c + 2);
            if (rc) break;
        }
    }
    if (rc || truncated) { // drain, then report / fall back to the exact single-shot semantics
        cudaStreamSynchronize(e->s_h2d);
        cudaStreamSynchronize(e->s_d2h);
        if (pump) pump->abort(rc ? rc : DBEEL_ERR_INVALID_ARG); // its threads are joined when it goes out of scope
        return rc ? rc : kFallbackSingleShot;
    }
    if (sh.bloom_file) {
        CU(cudaStreamWaitEvent(e->s_d2h, e->ev_comp[(np - 1) & 1], 0));
        CU(cudaMemcpyAsync(io ? (void *)e->pin_bloom : out->bloom, e->bloom_dev, sh.bloom_file, cudaMemcpyDeviceToHost, e->s_d2h));
    }
    CU(cudaStreamSynchronize(e->s_d2h));
    CU(cudaStreamSynchronize(e->s_h2d));
    if (io) {
        if (sh.bloom_file) {
            const int wrc = io->write(io->ctx, DBEEL_STREAM_BLOOM, 0, e->pin_bloom, sh.bloom_file);
            if (wrc) return fail(e, wrc, "stream write callback failed (.bloom)");
        }
        const int frc = pump->finish(); // every partition's bytes have gone through the write callback
        if (frc) return fail(e, frc, "stream write callback failed");
    }
    if (trace) {
        fprintf(stderr, "[dbeel trace] %u partitions; ms since the first H2D began: h2d[begin,end] kernels[begin,end] d2h[begin,end]\n", np);
        for (uint32_t c = 0; c < np; c++) {
            float t[6];
            for (int k = 0; k < 6; k++) cudaEventElapsedTime(&t[k], tev[0], tev[6 * c + k]);
            fprintf(stderr, "[dbeel trace] p%02u h2d %6.2f %6.2f  kernels %6.2f %6.2f  d2h %6.2f %6.2f\n", c, t[0], t[1], t[2], t[3], t[4], t[5]);
        }
        for (auto &ev : tev) cudaEventDestroy(ev);
    }
    out->data_len = out_data;
    out->items_written = out_items;
    out->index_len = out_items * 16;
    out->bloom_len = sh.bloom_file;
    total.entries_out = out_items;
    total.output_bytes = out->data_len + out->index_len + out->bloom_len;
    total.kernel_launches += sh.bloom_file ? 1 : 0;
    total.partitions = np;
    e->stats = total;
    return DBEEL_OK;
}

// The host form of a device-resident job (dbeel_compact below the pipeline, dbeel_flush_many, dbeel_compact_many): the runs
// go down into stage_in, run_job_device writes into `dout` (from stage_outputs), and what it wrote comes back into `out`, the
// filter as bloom_len bytes.  ms_h2d / ms_d2h time the two copies.
int run_job_staged(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *o, bool flush, dbeel_out *dout,
                   uint64_t bloom_len, dbeel_out *out, const JobExtra *ex = nullptr) {
    cudaStream_t s = e->stream;
    std::vector<HostPiece> pieces;
    for (uint32_t r = 0; r < n_runs; r++) {
        pieces.push_back(HostPiece{runs[r].data, runs[r].data_len, nullptr});
        pieces.push_back(HostPiece{runs[r].index, runs[r].index_len, nullptr});
    }
    CU(cudaEventRecord(e->ev[EV_H2D0], s));
    int rc = stage_host(e, pieces);
    if (rc) return rc;
    CU(cudaEventRecord(e->ev[EV_H2D1], s));
    std::vector<dbeel_run> dr(n_runs);
    for (uint32_t r = 0; r < n_runs; r++) dr[r] = dbeel_run{pieces[2 * r].dev, runs[r].data_len, pieces[2 * r + 1].dev, runs[r].index_len};
    if ((rc = run_job_device(e, dr.data(), n_runs, o, flush, dout, ex))) return rc;
    CU(cudaEventRecord(e->ev[EV_D2H0], s));
    if ((rc = copy_back(e, *dout, bloom_len, out))) return rc;
    CU(cudaEventRecord(e->ev[EV_D2H1], s));
    CU(cudaStreamSynchronize(s));
    cudaEventElapsedTime(&e->stats.ms_h2d, e->ev[EV_H2D0], e->ev[EV_H2D1]);
    cudaEventElapsedTime(&e->stats.ms_d2h, e->ev[EV_D2H0], e->ev[EV_D2H1]);
    return DBEEL_OK;
}

// host buffers in / out around run_job_device
int run_job_host(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *o, bool flush,
                 dbeel_out *out) {
    JobShape sh;
    shape_of(runs, n_runs, o, flush, &sh);
    if (n_runs > DBEEL_MAX_RUNS) return fail(e, DBEEL_ERR_TOO_MANY_RUNS, "too many runs");
    if (out->data_cap < sh.data_total || out->index_cap < sh.n_total * 16 || out->bloom_cap < sh.bloom_file)
        return fail(e, DBEEL_ERR_CAPACITY, "output buffer smaller than dbeel_compact_bound");
    for (uint32_t r = 0; r < n_runs; r++)
        if ((runs[r].data_len && !runs[r].data) || (runs[r].index_len && !runs[r].index))
            return fail(e, DBEEL_ERR_INVALID_ARG, "null run buffer");
    if (e->pipeline && !flush && !(o->flags & DBEEL_FLAG_VERIFY_SORTED) && sh.n_total < 0xFFFFFFFEull &&
        sh.data_total + sh.index_total >= e->pipeline_min_bytes) {
        int prc = run_job_host_pipelined(e, runs, n_runs, o, out, sh);
        if (prc != kFallbackSingleShot) return prc;
        out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    }

    dbeel_out dout;
    const int rc = stage_outputs(e, sh.data_total, sh.n_total * 16, sh.bloom_file, &dout);
    return rc ? rc : run_job_staged(e, runs, n_runs, o, flush, &dout, sh.bloom_file, out);
}

// ------------------------------------------------------------------------------------ N3: the storage edge
// dbeel_compact_stream for a job the pipeline does not take (too small to partition, an index the planner does not trust,
// a run that ended early): every file whole into page-locked memory, the single-shot host path, the outputs whole through
// the write callback -- the exact semantics of dbeel_compact, the callbacks just replace the caller's buffers.
struct HostBlock {
    uint8_t *p = nullptr;
    ~HostBlock() { if (p) cudaFreeHost(p); }
    bool alloc(uint64_t n) {
        if (cudaHostAlloc(reinterpret_cast<void **>(&p), n ? n : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); p = nullptr; }
        return p != nullptr;
    }
};

int run_job_stream_whole(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *o, const dbeel_stream_io *io,
                         dbeel_out *out, const JobShape &sh) {
    std::vector<uint64_t> doff(n_runs), ioff(n_runs);
    uint64_t pos = 0;
    for (uint32_t r = 0; r < n_runs; r++) {
        doff[r] = pos;
        pos += align_up(runs[r].data_len + 16, kAlign);
        ioff[r] = pos;
        pos += align_up(runs[r].index_len + 16, kAlign);
    }
    HostBlock in, ob;
    if (!in.alloc(pos)) return fail(e, DBEEL_ERR_NOMEM, "cudaHostAlloc(stream inputs)");
    std::vector<StreamPump::ReadTask> rt;
    std::vector<dbeel_run> hr(n_runs);
    for (uint32_t r = 0; r < n_runs; r++) {
        hr[r] = dbeel_run{in.p + doff[r], runs[r].data_len, in.p + ioff[r], runs[r].index_len};
        for (uint64_t d = 0; d < runs[r].data_len; d += StreamPump::kPiece)
            rt.push_back(StreamPump::ReadTask{0, r, DBEEL_STREAM_DATA, d, std::min<uint64_t>(StreamPump::kPiece, runs[r].data_len - d), in.p + doff[r] + d});
        for (uint64_t d = 0; d < runs[r].index_len; d += StreamPump::kPiece)
            rt.push_back(StreamPump::ReadTask{0, r, DBEEL_STREAM_INDEX, d, std::min<uint64_t>(StreamPump::kPiece, runs[r].index_len - d), in.p + ioff[r] + d});
    }
    int rc = parallel_pieces(rt.size(), [&](size_t k) { return io->read(io->ctx, rt[k].run, rt[k].kind, rt[k].off, rt[k].len, rt[k].dst); });
    if (rc) return fail(e, rc, "stream read callback failed");
    const uint64_t dc = sh.data_total, ic = sh.n_total * 16, bc = sh.bloom_file;
    const uint64_t o_index = align_up(dc + 16, kAlign), o_bloom = o_index + align_up(ic + 16, kAlign);
    if (!ob.alloc(o_bloom + align_up(bc + 16, kAlign))) return fail(e, DBEEL_ERR_NOMEM, "cudaHostAlloc(stream outputs)");
    dbeel_out o2 = {ob.p, dc, 0, ob.p + o_index, ic, 0, bc ? ob.p + o_bloom : nullptr, bc, 0, 0};
    const int saved = e->pipeline;
    e->pipeline = 0;
    rc = run_job_host(e, hr.data(), n_runs, o, false, &o2);
    e->pipeline = saved;
    if (rc) return rc;
    struct WTask { uint32_t kind; uint64_t off, len; const uint8_t *src; };
    std::vector<WTask> wt;
    for (uint64_t d = 0; d < o2.data_len; d += StreamPump::kPiece)
        wt.push_back(WTask{DBEEL_STREAM_DATA, d, std::min<uint64_t>(StreamPump::kPiece, o2.data_len - d), ob.p + d});
    for (uint64_t d = 0; d < o2.index_len; d += StreamPump::kPiece)
        wt.push_back(WTask{DBEEL_STREAM_INDEX, d, std::min<uint64_t>(StreamPump::kPiece, o2.index_len - d), ob.p + o_index + d});
    if (o2.bloom_len) wt.push_back(WTask{DBEEL_STREAM_BLOOM, 0, o2.bloom_len, ob.p + o_bloom});
    rc = parallel_pieces(wt.size(), [&](size_t k) { return io->write(io->ctx, wt[k].kind, wt[k].off, wt[k].src, wt[k].len); });
    if (rc) return fail(e, rc, "stream write callback failed");
    out->data_len = o2.data_len;
    out->index_len = o2.index_len;
    out->bloom_len = o2.bloom_len;
    out->items_written = o2.items_written;
    return DBEEL_OK;
}

int stream_entry(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts, const dbeel_stream_io *io,
                 dbeel_out *out) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || !io || !io->read || !io->write || (n_runs && !runs)) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    const Claim c(e);
    if (c.rc) return c.rc;
    dbeel_compact_opts o;
    default_opts(&o);
    if (opts) o = *opts;
    if (!(o.bloom_fp > 0.0 && o.bloom_fp < 1.0)) return fail(e, DBEEL_ERR_INVALID_ARG, "bloom_fp must be in (0,1)");
    if (n_runs > DBEEL_MAX_RUNS) return fail(e, DBEEL_ERR_TOO_MANY_RUNS, "too many runs");
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    JobShape sh;
    shape_of(runs, n_runs, &o, false, &sh);
    if (e->pipeline && !(o.flags & DBEEL_FLAG_VERIFY_SORTED) && sh.n_total < 0xFFFFFFFEull &&
        sh.data_total + sh.index_total >= e->pipeline_min_bytes) {
        const int prc = run_job_host_pipelined(e, runs, n_runs, &o, out, sh, io);
        if (prc != kFallbackSingleShot) return prc;
        out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    }
    return run_job_stream_whole(e, runs, n_runs, &o, io, out, sh);
}

int entry(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts, dbeel_out *out,
          bool flush, bool device) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || (n_runs && !runs)) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    const Claim c(e);
    if (c.rc) return c.rc;
    dbeel_compact_opts o;
    default_opts(&o);
    if (opts) o = *opts;
    if (!(o.bloom_fp > 0.0 && o.bloom_fp < 1.0)) return fail(e, DBEEL_ERR_INVALID_ARG, "bloom_fp must be in (0,1)");
    return device ? run_job_device(e, runs, n_runs, &o, flush, out) : run_job_host(e, runs, n_runs, &o, flush, out);
}


// ------------------------------------------------------------------------------------ N2: batched point lookups

constexpr uint64_t kBloomTrailer = 8 + 8 + 4 + 144; // nbits, bitmap_bits, k_num, 2 x SipHasher13 (9 x u64 each)

inline uint64_t rd64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
inline uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }

// head = the file's first 8 bytes, tail = its last kBloomTrailer bytes (both in host memory)
int parse_bloom(dbeel_engine *e, const uint8_t *head, const uint8_t *tail, uint64_t file_len, TableDesc *t) {
    const uint64_t n_words = rd64(head);
    if (n_words > (1ull << 40) || file_len != 8 + 4 * n_words + kBloomTrailer) return fail(e, DBEEL_ERR_BAD_BLOOM, "bloom file length does not match its word count");
    t->bits = rd64(tail + 8); // Bloom.bitmap_bits (the BitVec's own nbits precedes it)
    t->k_num = rd32(tail + 16);
    if (t->bits < 2 || t->bits > 32 * n_words || t->k_num == 0) return fail(e, DBEEL_ERR_BAD_BLOOM, "bloom parameters out of range");
    t->bits_magic = (uint64_t)((((unsigned __int128)1) << 64) / t->bits);
    for (int h = 0; h < 2; h++) { // SipHasher13 { k0, k1, length, state { v0, v2, v1, v3 }, tail, ntail }
        t->sip[2 * h] = rd64(tail + 20 + 72 * h);
        t->sip[2 * h + 1] = rd64(tail + 20 + 72 * h + 8);
    }
    return DBEEL_OK;
}

// The argument checks of both batched reads (dbeel_get_many*, dbeel_get_values*), before the engine is taken.
int lookup_args(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const uint64_t *key_off, uint64_t n_keys,
                uint32_t mode, const dbeel_lookup_result *results) {
    if ((n_tables && !tables) || (n_keys && (!key_off || !results))) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (mode > DBEEL_LOOKUP_EXACT) return fail(e, DBEEL_ERR_INVALID_ARG, "unknown lookup mode");
    if (n_tables > 65536) return fail(e, DBEEL_ERR_TOO_MANY_RUNS, "more than 65536 tables");
    return DBEEL_OK;
}

// The tables as k_lookup reads them, shared by both batched reads: table checks, the bloom trailers parsed on the host and,
// for host callers, the tables, keys and offsets staged into stage_in (the device path reads only each trailer back).  The
// TableDesc array goes down from the pinned block into `d_desc`; the pinned block is at least `pin_min` bytes.
int stage_lookup(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys, const uint64_t *key_off,
                 uint64_t n_keys, bool device, uint64_t pin_min, TableDesc *d_desc, const uint8_t **d_keys, const uint64_t **d_off) {
    cudaStream_t s = e->stream;
    for (uint32_t i = 0; i < n_tables; i++) {
        const dbeel_table &t = tables[i];
        if (t.index_len % DBEEL_INDEX_ENTRY_SIZE) return fail(e, DBEEL_ERR_INVALID_ARG, "index length is not a multiple of 16");
        if ((t.data_len && !t.data) || (t.index_len && !t.index) || (t.bloom_len && !t.bloom)) return fail(e, DBEEL_ERR_INVALID_ARG, "null table buffer");
        if (t.bloom_len && (t.bloom_len < 8 + kBloomTrailer || (t.bloom_len - 8 - kBloomTrailer) % 4))
            return fail(e, DBEEL_ERR_BAD_BLOOM, "bloom file length is not 8 + 4 * words + 164");
        if (device && (((uintptr_t)t.index & 15) || ((uintptr_t)t.bloom & 3))) return fail(e, DBEEL_ERR_INVALID_ARG, "misaligned device buffer");
    }
    std::vector<TableDesc> td(n_tables);
    *d_keys = static_cast<const uint8_t *>(keys);
    *d_off = key_off;
    int rc = ensure_pinned(e, std::max<uint64_t>({4096, pin_min, (uint64_t)n_tables * (8 + kBloomTrailer) + n_tables * sizeof(TableDesc)}));
    if (rc) return rc;
    uint8_t *pin_desc = e->pin + (uint64_t)n_tables * (8 + kBloomTrailer);
    if (device) {
        for (uint32_t i = 0; i < n_tables; i++) {
            const dbeel_table &t = tables[i];
            td[i] = TableDesc{static_cast<const uint8_t *>(t.data), t.data_len, static_cast<const uint4 *>(t.index),
                              t.index_len / DBEEL_INDEX_ENTRY_SIZE, nullptr, 0, 0, 0, 0, {0, 0, 0, 0}};
            if (!t.bloom_len) continue;
            const uint8_t *b = static_cast<const uint8_t *>(t.bloom);
            uint8_t *hp = e->pin + (uint64_t)i * (8 + kBloomTrailer);
            CU(cudaMemcpyAsync(hp, b, 8, cudaMemcpyDeviceToHost, s));
            CU(cudaMemcpyAsync(hp + 8, b + t.bloom_len - kBloomTrailer, kBloomTrailer, cudaMemcpyDeviceToHost, s));
            td[i].words = reinterpret_cast<const uint32_t *>(b + 8);
        }
        CU(cudaStreamSynchronize(s));
        for (uint32_t i = 0; i < n_tables; i++)
            if (tables[i].bloom_len) {
                const uint8_t *hp = e->pin + (uint64_t)i * (8 + kBloomTrailer);
                if ((rc = parse_bloom(e, hp, hp + 8, tables[i].bloom_len, &td[i]))) return rc;
            }
    } else { // host buffers: the tables, the keys and the offsets go down
        if (!keys && key_off[n_keys]) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
        std::vector<HostPiece> pieces{{keys, key_off[n_keys], nullptr}, {key_off, (n_keys + 1) * 8, nullptr}};
        for (uint32_t i = 0; i < n_tables; i++) {
            const dbeel_table &t = tables[i];
            pieces.insert(pieces.end(), {{t.data, t.data_len, nullptr}, {t.index, t.index_len, nullptr}, {t.bloom, t.bloom_len, nullptr}});
        }
        if ((rc = stage_host(e, pieces))) return rc;
        *d_keys = pieces[0].dev;
        *d_off = reinterpret_cast<const uint64_t *>(pieces[1].dev);
        for (uint32_t i = 0; i < n_tables; i++) {
            const dbeel_table &t = tables[i];
            const HostPiece *tp = &pieces[2 + 3 * i];
            td[i] = TableDesc{tp[0].dev, t.data_len, reinterpret_cast<const uint4 *>(tp[1].dev), t.index_len / DBEEL_INDEX_ENTRY_SIZE, nullptr, 0, 0, 0, 0, {0, 0, 0, 0}};
            if (!t.bloom_len) continue;
            const uint8_t *b = static_cast<const uint8_t *>(t.bloom);
            if ((rc = parse_bloom(e, b, b + t.bloom_len - kBloomTrailer, t.bloom_len, &td[i]))) return rc;
            td[i].words = reinterpret_cast<const uint32_t *>(tp[2].dev + 8);
        }
    }
    if (n_tables) {
        memcpy(pin_desc, td.data(), n_tables * sizeof(TableDesc));
        CU(cudaMemcpyAsync(d_desc, pin_desc, n_tables * sizeof(TableDesc), cudaMemcpyHostToDevice, s));
    }
    return DBEEL_OK;
}

int lookup_entry(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys, const uint64_t *key_off,
                 uint64_t n_keys, uint32_t mode, dbeel_lookup_result *results, bool device) {
    static_assert(sizeof(dbeel_lookup_result) == 16, "result rows are written as uint4");
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (const int arc = lookup_args(e, tables, n_tables, key_off, n_keys, mode, results)) return arc;
    const Claim c(e);
    if (c.rc) return c.rc;
    if (n_keys == 0) return DBEEL_OK;
    cudaStream_t s = e->stream;
    int rc = ensure_device(e, &e->ws, &e->ws_cap, std::max<uint64_t>(4096, n_tables * sizeof(TableDesc)));
    dbeel_out rows; // host callers: the rows before their D2H
    if (!rc && !device) rc = stage_outputs(e, n_keys * 16, 0, 0, &rows);
    if (rc) return rc;
    const uint8_t *d_keys;
    const uint64_t *d_off;
    if ((rc = stage_lookup(e, tables, n_tables, keys, key_off, n_keys, device, 0, reinterpret_cast<TableDesc *>(e->ws), &d_keys, &d_off)))
        return rc;
    uint4 *d_res = reinterpret_cast<uint4 *>(device ? results : rows.data);
    LookupParams lp{reinterpret_cast<const TableDesc *>(e->ws), n_tables, mode, d_keys, d_off, n_keys, d_res};
    CU(cudaEventRecord(e->ev[EV_START], s));
    k_lookup<<<(uint32_t)((n_keys + 255) / 256), 256, 0, s>>>(lp);
    CU(cudaGetLastError());
    CU(cudaEventRecord(e->ev[EV_GATHER], s));
    if (!device) CU(cudaMemcpyAsync(results, d_res, n_keys * 16, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaEventElapsedTime(&e->stats.ms_total, e->ev[EV_START], e->ev[EV_GATHER]));
    e->stats.kernel_launches = 1;
    e->stats.entries_in = n_keys;
    return DBEEL_OK;
}


// ------------------------------------------------------------------------------------ cfg5: shard routing

// batch / out_index / shard_of are device pointers; ring, counts, bytes live in host memory.
int route_entry(dbeel_engine *e, const dbeel_run *batch, const uint32_t *ring, uint32_t n_shards, void *out_index, uint64_t out_index_cap,
                uint32_t *shard_of, void *out_hash64, uint64_t *counts, uint64_t *bytes) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!batch || !ring || !counts || n_shards == 0) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (n_shards > kRouteMaxShards) return fail(e, DBEEL_ERR_INVALID_ARG, "more shards than DBEEL_MAX_SHARDS");
    for (uint32_t s = 1; s < n_shards; s++)
        if (ring[s - 1] >= ring[s]) return fail(e, DBEEL_ERR_INVALID_ARG, "ring hashes must be strictly ascending");
    const Claim c(e);
    if (c.rc) return c.rc;
    const uint64_t n64 = batch->index_len / DBEEL_INDEX_ENTRY_SIZE;
    for (uint32_t s = 0; s < n_shards; s++) { counts[s] = 0; if (bytes) bytes[s] = 0; }
    if (n64 >= 0xFFFFFFF0ull) return fail(e, DBEEL_ERR_TOO_MANY_ENTRIES, "too many arrivals in one batch");
    if (n64 == 0) return DBEEL_OK;
    if (out_index_cap < n64 * 16 || !out_index) return fail(e, DBEEL_ERR_CAPACITY, "routed index buffer too small");
    if (((uintptr_t)batch->index | (uintptr_t)out_index) & 15) return fail(e, DBEEL_ERR_INVALID_ARG, "index buffers must be 16-byte aligned");
    RouteParams p;
    p.data = static_cast<const uint8_t *>(batch->data);
    p.data_len = batch->data_len;
    p.index = static_cast<const uint4 *>(batch->index);
    p.n = (uint32_t)n64;
    p.n_shards = n_shards;
    p.n_blocks = (p.n + kRouteThreads - 1) / kRouteThreads;
    uint64_t off = 0;
    const uint64_t o_ring = carve_ws(&off, 4ull * n_shards), o_tot = carve_ws(&off, 8ull * (3 * n_shards + 1));
    const uint64_t o_hist = carve_ws(&off, 4ull * p.n_blocks * n_shards), o_owner = carve_ws(&off, shard_of ? 0 : 4ull * p.n);
    const uint64_t o_h64 = carve_ws(&off, out_hash64 ? 8ull * p.n : 0);
    int rc = ensure_device(e, &e->route_ws, &e->route_ws_cap, off);
    if (!rc) rc = ensure_pinned(e, 4096 + 8ull * (3 * n_shards + 1));
    if (rc) return rc;
    cudaStream_t s = e->stream;
    // the ring goes down through the mapped pinned block like every small header (no copy-engine traffic on this stream)
    memcpy(e->pin, ring, 4ull * n_shards);
    p.ring = reinterpret_cast<const uint32_t *>(e->route_ws + o_ring);
    p.totals = reinterpret_cast<unsigned long long *>(e->route_ws + o_tot);
    p.hist = reinterpret_cast<uint32_t *>(e->route_ws + o_hist);
    p.shard_of = shard_of ? shard_of : reinterpret_cast<uint32_t *>(e->route_ws + o_owner);
    p.out_index = static_cast<uint4 *>(out_index);
    p.hash64 = out_hash64 ? reinterpret_cast<unsigned long long *>(e->route_ws + o_h64) : nullptr;
    p.out_hash64 = static_cast<unsigned long long *>(out_hash64);
    CU(cudaEventRecord(e->ev[EV_START], s));
    k_copy_words<<<(n_shards + 255) / 256, 256, 0, s>>>(reinterpret_cast<uint32_t *>(e->route_ws + o_ring), reinterpret_cast<const uint32_t *>(e->pin_dev), n_shards);
    CU(cudaMemsetAsync(p.totals, 0, 8ull * 3 * n_shards, s));
    CU(cudaMemsetAsync(p.totals + 3 * n_shards, 0xFF, 8, s));
    k_route_hash<<<p.n_blocks, kRouteThreads, 0, s>>>(p);
    k_route_scan<<<n_shards, 1024, 0, s>>>(p);
    unsigned long long *host_tot = reinterpret_cast<unsigned long long *>(e->pin + 4096);
    k_route_starts<<<1, 256, 0, s>>>(p, reinterpret_cast<unsigned long long *>(e->pin_dev + 4096));
    k_route_scatter<<<p.n_blocks, kRouteThreads, 0, s>>>(p);
    CU(cudaEventRecord(e->ev[EV_GATHER], s));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));
    dbeel_stats &st = e->stats;
    st.entries_in = n64;
    st.kernel_launches = 5;
    cudaEventElapsedTime(&st.ms_total, e->ev[EV_START], e->ev[EV_GATHER]);
    if (host_tot[3 * n_shards] != ~0ull) return fail(e, DBEEL_ERR_INVALID_ARG, "an arrival's index record does not frame an entry inside .data");
    for (uint32_t k = 0; k < n_shards; k++) {
        counts[k] = host_tot[k];
        if (bytes) bytes[k] = host_tot[n_shards + k];
    }
    st.entries_out = n64;
    st.input_bytes = n64 * 16;
    return DBEEL_OK;
}

// key_hash64: device; stream_starts / cuts / cut_starts: host
int cuts_entry(dbeel_engine *e, const void *key_hash64, const uint64_t *stream_starts, uint32_t n_streams, uint32_t capacity,
               uint32_t *cuts, uint32_t *cut_starts, uint32_t max_cuts_total) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!stream_starts || !cuts || !cut_starts || !n_streams) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (capacity < 1 || capacity > kCutMaxCapacity) return fail(e, DBEEL_ERR_INVALID_ARG, "capacity above what the device cut supports (use dbeel_memtable_cut)");
    const Claim c(e);
    if (c.rc) return c.rc;
    // a stream of n arrivals has at most n / capacity full memtables
    std::vector<uint32_t> base(n_streams + 1, 0);
    for (uint32_t s = 0; s < n_streams; s++) {
        if (stream_starts[s + 1] < stream_starts[s] || stream_starts[s + 1] - stream_starts[s] >= 0xFFFFFFF0ull)
            return fail(e, DBEEL_ERR_INVALID_ARG, "stream_starts must ascend");
        base[s + 1] = base[s] + (uint32_t)((stream_starts[s + 1] - stream_starts[s]) / capacity);
    }
    const uint32_t total_max = base[n_streams];
    for (uint32_t s = 0; s <= n_streams; s++) cut_starts[s] = 0;
    if (stream_starts[n_streams] == stream_starts[0]) return DBEEL_OK;
    if (!key_hash64) return fail(e, DBEEL_ERR_INVALID_ARG, "null key identities");
    uint64_t off = 0;
    const uint64_t o_starts = carve_ws(&off, 8ull * (n_streams + 1)), o_base = carve_ws(&off, 4ull * n_streams), o_n = carve_ws(&off, 4ull * n_streams);
    const uint64_t o_cuts = carve_ws(&off, 4ull * (total_max + 1));
    const uint64_t hdr = o_n; // starts | base go down, n_cuts | cuts come back
    int rc = ensure_device(e, &e->route_ws, &e->route_ws_cap, off);
    if (!rc) rc = ensure_pinned(e, off);
    if (rc) return rc;
    memcpy(e->pin + o_starts, stream_starts, 8ull * (n_streams + 1));
    memcpy(e->pin + o_base, base.data(), 4ull * n_streams);
    cudaStream_t s = e->stream;
    CU(cudaEventRecord(e->ev[EV_START], s));
    k_copy_words<<<(uint32_t)((hdr / 4 + 255) / 256), 256, 0, s>>>(reinterpret_cast<uint32_t *>(e->route_ws), reinterpret_cast<const uint32_t *>(e->pin_dev),
                                                                    (uint32_t)(hdr / 4));
    CutParams p;
    p.hash64 = static_cast<const unsigned long long *>(key_hash64);
    p.starts = reinterpret_cast<const unsigned long long *>(e->route_ws + o_starts);
    p.n_streams = n_streams;
    p.capacity = capacity;
    p.max_cuts = total_max;
    p.cut_base = reinterpret_cast<const uint32_t *>(e->route_ws + o_base);
    p.cuts = reinterpret_cast<uint32_t *>(e->route_ws + o_cuts);
    p.n_cuts = reinterpret_cast<uint32_t *>(e->route_ws + o_n);
    k_memtable_cuts<<<n_streams, 1024, 12ull * kCutSlots, s>>>(p);
    k_publish<<<1, 256, 0, s>>>(reinterpret_cast<uint32_t *>(e->pin_dev + o_n), p.n_cuts, n_streams, reinterpret_cast<uint32_t *>(e->pin_dev + o_cuts),
                                p.cuts, total_max);
    CU(cudaEventRecord(e->ev[EV_GATHER], s));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));
    dbeel_stats &st = e->stats;
    st.kernel_launches = 3;
    st.entries_in = stream_starts[n_streams] - stream_starts[0];
    cudaEventElapsedTime(&st.ms_total, e->ev[EV_START], e->ev[EV_GATHER]);
    const uint32_t *hn = reinterpret_cast<const uint32_t *>(e->pin + o_n), *hc = reinterpret_cast<const uint32_t *>(e->pin + o_cuts);
    uint32_t w = 0;
    for (uint32_t k = 0; k < n_streams; k++) {
        cut_starts[k] = w;
        const uint32_t nc = hn[k] < base[k + 1] - base[k] ? hn[k] : base[k + 1] - base[k];
        if (w + nc > max_cuts_total) return fail(e, DBEEL_ERR_CAPACITY, "cuts array too small");
        for (uint32_t c = 0; c < nc; c++) cuts[w++] = hc[base[k] + c];
    }
    cut_starts[n_streams] = w;
    return DBEEL_OK;
}

// ------------------------------------------------------------------------------------ N4: WAL replay + flush

int wal_flush_entry(dbeel_engine *e, const void *wal, uint64_t wal_len, uint32_t capacity, dbeel_out *out, bool device) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || (wal_len && !wal)) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    const Claim c(e);
    if (c.rc) return c.rc;
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    const uint64_t n_pages64 = (wal_len + kWalPage - 1) / kWalPage;
    if (n_pages64 >= 0xFFFFFFF0ull) return fail(e, DBEEL_ERR_TOO_MANY_ENTRIES, "write-ahead log too large");
    if (wal_len == 0) return DBEEL_OK;
    cudaStream_t s = e->stream;
    const uint32_t n_pages = (uint32_t)n_pages64, nodes = n_pages + 1;
    uint32_t levels = 0;
    while ((1ull << levels) < nodes) levels++;

    const uint8_t *d_wal = static_cast<const uint8_t *>(wal);
    float ms_h2d = 0;
    if (!device) { // host log: stage it down (the flush below writes into staging too)
        std::vector<HostPiece> log{{wal, wal_len, nullptr}};
        CU(cudaEventRecord(e->ev[EV_H2D0], s));
        if (const int rc = stage_host(e, log)) return rc;
        CU(cudaEventRecord(e->ev[EV_H2D1], s));
        d_wal = log[0].dev;
    } else if ((uintptr_t)wal & 15) {
        return fail(e, DBEEL_ERR_INVALID_ARG, "device log buffer must be 16-byte aligned");
    }
    // scratch: jump / cnt tables, per-page sizes, the arrival index, 3 totals
    uint64_t off = 0;
    const uint64_t o_jump = carve_ws(&off, 4ull * (levels + 1) * nodes), o_cnt = carve_ws(&off, 4ull * (levels + 1) * nodes);
    const uint64_t o_sizes = carve_ws(&off, 8ull * n_pages), o_index = carve_ws(&off, 16ull * n_pages), o_tot = carve_ws(&off, 32);
    int rc = ensure_device(e, &e->wal_ws, &e->wal_ws_cap, off);
    if (!rc) rc = ensure_pinned(e, 4096);
    if (rc) return rc;
    WalParams w;
    w.wal = d_wal;
    w.len = wal_len;
    w.n_pages = n_pages;
    w.levels = levels;
    w.jump = reinterpret_cast<uint32_t *>(e->wal_ws + o_jump);
    w.cnt = reinterpret_cast<uint32_t *>(e->wal_ws + o_cnt);
    w.sizes = reinterpret_cast<uint2 *>(e->wal_ws + o_sizes);
    w.index = reinterpret_cast<uint4 *>(e->wal_ws + o_index);
    w.totals = reinterpret_cast<unsigned long long *>(e->wal_ws + o_tot);
    CU(cudaMemsetAsync(w.totals, 0, 32, s));
    const uint32_t grid = (nodes + 255) / 256;
    k_wal_parse<<<grid, 256, 0, s>>>(w);
    for (uint32_t k = 0; k < levels; k++) k_wal_double<<<grid, 256, 0, s>>>(w, k);
    k_wal_select<<<(n_pages + 255) / 256, 256, 0, s>>>(w);
    k_publish<<<1, 256, 0, s>>>(reinterpret_cast<uint32_t *>(e->pin_dev), reinterpret_cast<const uint32_t *>(w.totals), 6,
                                nullptr, nullptr, 0);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));
    if (!device) cudaEventElapsedTime(&ms_h2d, e->ev[EV_H2D0], e->ev[EV_H2D1]);
    unsigned long long totals[3];
    memcpy(totals, e->pin, sizeof totals);
    const uint64_t n_rec = totals[0], bytes = totals[1];
    const uint32_t wal_launches = levels + 3;
    if (totals[2] & kWalTooLarge) return fail(e, DBEEL_ERR_ITEM_TOO_LARGE, "a logged entry exceeds u32::MAX bytes");
    if (n_rec == 0) { e->stats.kernel_launches = wal_launches; return DBEEL_OK; }

    // ---- the flush: the log is the batch's .data, the selected records its (sparse) .index
    dbeel_compact_opts o;
    default_opts(&o);
    JobExtra ex;
    ex.sparse_offsets = true;
    ex.data_bytes = bytes;
    dbeel_run batch{d_wal, wal_len, w.index, n_rec * 16};
    if (out->data_cap < bytes || out->index_cap < n_rec * 16) return fail(e, DBEEL_ERR_CAPACITY, "output buffer too small for the replayed entries");
    if (device) {
        rc = run_job_device(e, &batch, 1, &o, true, out, &ex);
    } else {
        dbeel_out dout = {};
        rc = stage_outputs(e, bytes, n_rec * 16, 0, &dout);
        if (!rc) rc = run_job_device(e, &batch, 1, &o, true, &dout, &ex);
        if (!rc && dout.items_written <= capacity) {
            rc = copy_back(e, dout, 0, out);
            CU(cudaStreamSynchronize(s));
        }
        out->data_len = dout.data_len;
        out->index_len = dout.index_len;
        out->items_written = dout.items_written;
        e->stats.ms_h2d = ms_h2d;
    }
    if (rc) return rc;
    e->stats.kernel_launches += wal_launches;
    e->stats.input_bytes = wal_len;
    if (out->items_written > capacity) { // memtable.set(..)? -> ReachedCapacity (lsm_tree.rs:566, rbtree_arena lib.rs:458-461)
        out->data_len = out->index_len = out->items_written = 0;
        return fail(e, DBEEL_ERR_TREE_FULL, "the log holds more distinct keys than the memtable capacity");
    }
    return DBEEL_OK;
}


// ------------------------------------------------------------------------------------ N1: compact-many

struct JobShapes {
    std::vector<JobShape> shape;
    std::vector<uint64_t> bloom_off;
    uint64_t data = 0, index = 0, bloom = 0, entries = 0, runs = 0;
};

int job_shapes(dbeel_engine *e, const dbeel_job *jobs, uint32_t n_jobs, uint64_t bloom_min_size, double fp, JobShapes *js) {
    if (!(fp > 0.0 && fp < 1.0)) return e ? fail(e, DBEEL_ERR_INVALID_ARG, "bloom_fp must be in (0,1)") : DBEEL_ERR_INVALID_ARG;
    dbeel_compact_opts o;
    default_opts(&o);
    o.bloom_min_size = bloom_min_size;
    o.bloom_fp = fp;
    js->shape.assign(n_jobs, JobShape{});
    js->bloom_off.assign(n_jobs, 0);
    for (uint32_t g = 0; g < n_jobs; g++) {
        if (jobs[g].n_runs && !jobs[g].runs) return e ? fail(e, DBEEL_ERR_INVALID_ARG, "null run array") : DBEEL_ERR_INVALID_ARG;
        shape_of(jobs[g].runs, jobs[g].n_runs, &o, false, &js->shape[g]);
        js->data += js->shape[g].data_total;
        js->index += js->shape[g].n_total * 16;
        js->entries += js->shape[g].n_total;
        js->runs += jobs[g].n_runs;
        js->bloom_off[g] = js->bloom;
        js->bloom += align_up(js->shape[g].bloom_file, 16);
    }
    return DBEEL_OK;
}

int compact_many_entry(dbeel_engine *e, const dbeel_job *jobs, uint32_t n_jobs, uint64_t bloom_min_size, double fp, dbeel_out *out,
                       dbeel_job_result *results, bool device) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || (n_jobs && (!jobs || !results))) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    const Claim c(e);
    if (c.rc) return c.rc;
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    JobShapes js;
    int rc = job_shapes(e, jobs, n_jobs, bloom_min_size, fp, &js);
    if (rc) return rc;
    for (uint32_t g = 0; g < n_jobs; g++) results[g] = dbeel_job_result{0, 0, 0, 0, 0, 0, 0};
    if (js.runs > DBEEL_MAX_RUNS) return fail(e, DBEEL_ERR_TOO_MANY_RUNS, "more than DBEEL_MAX_RUNS runs over all jobs");
    if (js.entries >= 0xFFFFFFFEull) return fail(e, DBEEL_ERR_TOO_MANY_ENTRIES, "too many entries");
    if (out->data_cap < js.data || out->index_cap < js.index || out->bloom_cap < js.bloom)
        return fail(e, DBEEL_ERR_CAPACITY, "output buffer smaller than dbeel_compact_many_bound");
    if (n_jobs == 0 || js.entries == 0) return DBEEL_OK;
    cudaStream_t s = e->stream;

    // all runs back to back; host buffers are staged down first
    std::vector<dbeel_run> flat;
    std::vector<uint32_t> first(n_jobs + 1, 0);
    std::vector<int32_t> keep(n_jobs);
    for (uint32_t g = 0; g < n_jobs; g++) {
        first[g] = (uint32_t)flat.size();
        keep[g] = jobs[g].keep_tombstones;
        for (uint32_t r = 0; r < jobs[g].n_runs; r++) flat.push_back(jobs[g].runs[r]);
    }
    first[n_jobs] = (uint32_t)flat.size();
    dbeel_out dout = *out;
    if (!device) {
        for (auto &r : flat)
            if ((r.data_len && !r.data) || (r.index_len && !r.index)) return fail(e, DBEEL_ERR_INVALID_ARG, "null run buffer");
        if ((rc = stage_outputs(e, js.data, js.index, js.bloom, &dout))) return rc;
    } else if ((uintptr_t)out->bloom & 15) {
        return fail(e, DBEEL_ERR_INVALID_ARG, "device output buffers must be 16-byte aligned");
    }
    // per-job filters
    std::vector<BloomParams> bloom(n_jobs);
    for (uint32_t g = 0; g < n_jobs; g++) {
        bloom[g] = BloomParams{};
        const JobShape &sh = js.shape[g];
        if (!sh.bloom_file) continue;
        uint8_t seed[32];
        if (jobs[g].bloom_seed) {
            memcpy(seed, jobs[g].bloom_seed, 32);
        } else {
            FILE *f = fopen("/dev/urandom", "rb");
            if (!f || fread(seed, 1, 32, f) != 32) {
                if (f) fclose(f);
                return fail(e, DBEEL_ERR_INVALID_ARG, "no entropy source for the bloom seed");
            }
            fclose(f);
        }
        bloom[g].words = reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(dout.bloom) + js.bloom_off[g] + 8);
        bloom[g].bits = sh.bloom_bits;
        bloom[g].bits_magic = (uint64_t)((((unsigned __int128)1) << 64) / sh.bloom_bits);
        bloom[g].k_num = sh.bloom_k;
        for (int i = 0; i < 4; i++) memcpy(&bloom[g].sip[i], seed + 8 * i, 8);
    }
    if (js.bloom) CU(cudaMemsetAsync(dout.bloom, 0, js.bloom, s));
    dbeel_compact_opts o;
    default_opts(&o);
    o.bloom_min_size = bloom_min_size;
    o.bloom_fp = fp;
    JobExtra ex;
    ex.n_jobs = n_jobs;
    ex.job_first = first.data();
    ex.job_keep = keep.data();
    ex.job_bloom = bloom.data();
    ex.job_results = results;
    rc = device ? run_job_device(e, flat.data(), (uint32_t)flat.size(), &o, false, &dout, &ex)
                : run_job_staged(e, flat.data(), (uint32_t)flat.size(), &o, false, &dout, js.bloom, out, &ex);
    if (rc) return rc;
    for (uint32_t g = 0; g < n_jobs; g++) {
        results[g].bloom_off = js.bloom_off[g];
        results[g].bloom_len = js.shape[g].bloom_file;
    }
    out->data_len = dout.data_len;
    out->index_len = dout.index_len;
    out->bloom_len = js.bloom;
    out->items_written = dout.items_written;
    e->stats.output_bytes += js.bloom;
    return DBEEL_OK;
}

// ------------------------------------------------------------------------------------ N5: scans (iter_filter)

// the argument checks both scan entry points share; *key_bytes = the key ranges' bytes (0 for hash ranges)
int scan_args(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges, uint32_t n_ranges,
              const dbeel_job_result *results, const dbeel_scan_stop *stop, uint64_t *key_bytes) {
    if (!results || !stop || !ranges || (n_tables && !tables)) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (kind > DBEEL_SCAN_KEY) return fail(e, DBEEL_ERR_INVALID_ARG, "unknown scan kind");
    if (n_ranges == 0 || n_ranges > DBEEL_MAX_SCAN_RANGES) return fail(e, DBEEL_ERR_INVALID_ARG, "1 to DBEEL_MAX_SCAN_RANGES ranges");
    if (n_tables > DBEEL_MAX_RUNS) return fail(e, DBEEL_ERR_INVALID_ARG, "more than DBEEL_MAX_RUNS tables");
    const dbeel_key_ranges *kr = static_cast<const dbeel_key_ranges *>(ranges);
    *key_bytes = 0;
    if (kind == DBEEL_SCAN_KEY) {
        if (!kr->key_offsets) return fail(e, DBEEL_ERR_INVALID_ARG, "null key offsets");
        for (uint32_t k = 0; k < 2 * n_ranges; k++)
            if (kr->key_offsets[k + 1] < kr->key_offsets[k]) return fail(e, DBEEL_ERR_INVALID_ARG, "key offsets must ascend");
        *key_bytes = kr->key_offsets[2 * n_ranges] - kr->key_offsets[0];
        if (*key_bytes && !kr->keys) return fail(e, DBEEL_ERR_INVALID_ARG, "null range keys");
    }
    return DBEEL_OK;
}

// results and stop as a scan that delivered nothing leaves them
void clear_scan(dbeel_job_result *results, uint32_t nd, dbeel_scan_stop *stop) {
    for (uint32_t d = 0; d < nd; d++) results[d] = dbeel_job_result{0, 0, 0, 0, 0, 0, 0};
    *stop = dbeel_scan_stop{-1, DBEEL_SCAN_STOP_NONE, 0};
}

// ---- the ranges as the kernels read them (ScanParams.hash_ranges / key_off / keys), carved behind what the caller put
// at the front of the workspace.  land_ranges writes them into the pinned block at the same offsets and lands ws[0, bytes)
// -- the caller's front block included -- with one k_copy_words.
struct RangeHeader {
    uint64_t o_rng, o_keys, bytes;
};

RangeHeader carve_ranges(uint64_t *off, uint32_t kind, uint32_t nd, uint64_t key_bytes) {
    RangeHeader rh;
    rh.o_rng = carve_ws(off, kind == DBEEL_SCAN_KEY ? 8ull * (2 * nd + 1) : 8ull * nd);
    rh.o_keys = carve_ws(off, key_bytes + 16);
    rh.bytes = *off;
    return rh;
}

void land_ranges(dbeel_engine *e, const RangeHeader &rh, uint32_t kind, const void *ranges, uint32_t nd, uint64_t key_bytes,
                 ScanParams *sp) {
    uint8_t *ws = e->ws, *h = e->pin;
    if (kind == DBEEL_SCAN_KEY) {
        const dbeel_key_ranges *kr = static_cast<const dbeel_key_ranges *>(ranges);
        uint64_t *ko = reinterpret_cast<uint64_t *>(h + rh.o_rng);
        for (uint32_t k = 0; k <= 2 * nd; k++) ko[k] = kr->key_offsets[k] - kr->key_offsets[0];
        if (key_bytes) memcpy(h + rh.o_keys, static_cast<const uint8_t *>(kr->keys) + kr->key_offsets[0], key_bytes);
    } else {
        memcpy(h + rh.o_rng, ranges, 8ull * nd);
    }
    sp->key_kind = kind == DBEEL_SCAN_KEY ? 1u : 0u;
    sp->n_ranges = nd;
    sp->hash_ranges = reinterpret_cast<const uint32_t *>(ws + rh.o_rng);
    sp->key_off = reinterpret_cast<const unsigned long long *>(ws + rh.o_rng);
    sp->keys = ws + rh.o_keys;
    launch_k(e, k_copy_words, (uint32_t)((rh.bytes / 4 + 255) / 256), 256, 0, e->stream, reinterpret_cast<uint32_t *>(ws),
             reinterpret_cast<const uint32_t *>(e->pin_dev), (uint32_t)(rh.bytes / 4));
}

// ---- the split and phase 2 of a scan, shared by every call that returns entries
// Input: n 16-byte records {source address, 8 + klen, full_size} (ScanParams.flat) and a destination per record
// (ScanParams.dest, kScanNone = not delivered).  Output: the nd streams back to back, in record order inside each stream,
// every stream's .index offsets relative to its own first byte -- nd arrival batches.  split_emit runs it once, sized
// from a read-back (records may share .data bytes, so the output can be larger than the inputs); run_scan_plan runs it
// per partition, sized from the plan's bound.
struct SplitLayout {
    uint64_t o_ctl, o_memtab, header2_bytes; // second header, after the split is known: control block | (bytes, entries) before each stream
    uint64_t o_tot, o_dest, o_flat, o_split, o_hist, o_tbytes, o_tcount, o_cbytes, o_ccount, o_src;
    uint32_t n, nd, n_blocks;
};

SplitLayout carve_split(uint64_t *off, uint32_t n, uint32_t nd) {
    SplitLayout w;
    w.n = n;
    w.nd = nd;
    w.n_blocks = (n + kRouteThreads - 1) / kRouteThreads;
    const uint64_t res_tiles = (n + kResolveThreads - 1) / kResolveThreads, res_chunks = (res_tiles + 1023) / 1024;
    w.o_ctl = carve_ws(off, sizeof(Ctl));
    w.o_memtab = carve_ws(off, 16ull * (nd + 1));
    w.header2_bytes = *off - w.o_ctl;
    w.o_tot = carve_ws(off, 8ull * (3 * nd + 1));
    w.o_dest = carve_ws(off, 4ull * n);
    w.o_flat = carve_ws(off, 16ull * n);
    w.o_split = carve_ws(off, 16ull * n);
    w.o_hist = carve_ws(off, 4ull * w.n_blocks * nd);
    w.o_tbytes = carve_ws(off, 8 * res_tiles);
    w.o_tcount = carve_ws(off, 4 * res_tiles);
    w.o_cbytes = carve_ws(off, 8 * res_chunks);
    w.o_ccount = carve_ws(off, 4 * res_chunks);
    w.o_src = carve_ws(off, 8ull * n);
    return w;
}

// The split's workspace bound into the kernels' parameters: ScanParams' records, destinations and stop word (totals[3 nd],
// stop0 = none), the split's RouteParams and phase 2's workspace in Params.  n / n_blocks, tile_first, data_bound and the
// outputs are the caller's.
void split_bind(const SplitLayout &w, uint8_t *ws, ScanParams *sp, RouteParams *rp, Params *p) {
    sp->dest = reinterpret_cast<uint32_t *>(ws + w.o_dest);
    sp->flat = reinterpret_cast<uint4 *>(ws + w.o_flat);
    sp->stop = reinterpret_cast<unsigned long long *>(ws + w.o_tot) + 3ull * w.nd;
    sp->stop0 = ~0ull;
    *rp = RouteParams{};
    rp->index = sp->flat;
    rp->n_shards = w.nd;
    rp->shard_of = sp->dest;
    rp->hist = reinterpret_cast<uint32_t *>(ws + w.o_hist);
    rp->totals = reinterpret_cast<unsigned long long *>(ws + w.o_tot);
    rp->out_index = reinterpret_cast<uint4 *>(ws + w.o_split);
    memset(p, 0, sizeof *p);
    p->ctl = reinterpret_cast<Ctl *>(ws + w.o_ctl);
    p->tile_bytes = reinterpret_cast<unsigned long long *>(ws + w.o_tbytes);
    p->tile_count = reinterpret_cast<uint32_t *>(ws + w.o_tcount);
    p->chunk_bytes = reinterpret_cast<unsigned long long *>(ws + w.o_cbytes);
    p->chunk_count = reinterpret_cast<uint32_t *>(ws + w.o_ccount);
    p->src_ptr = reinterpret_cast<unsigned long long *>(ws + w.o_src);
    p->n_groups = w.nd;
    p->mem_table = reinterpret_cast<unsigned long long *>(ws + w.o_memtab);
}

// k_scan_hist drops what lies at or past the stop, k_route_scan / k_route_starts / k_route_scatter split the records
// stably into rp.out_index, and k_route_starts publishes the totals (counts | bytes | starts | stop, nd each + 1) to pub.
void launch_split(dbeel_engine *e, const ScanParams &sp, const RouteParams &rp, unsigned long long *pub) {
    cudaStream_t s = e->stream;
    launch_k(e, k_scan_hist, rp.n_blocks, kRouteThreads, 0, s, sp, rp);
    launch_k(e, k_route_scan, rp.n_shards, 1024, 0, s, rp);
    launch_k(e, k_route_starts, 1, 256, 0, s, rp, pub);
    launch_k(e, k_route_scatter, rp.n_blocks, kRouteThreads, 0, s, rp);
}

// Phase 2 over n split records (a bound: tiles past Ctl.span return at once): k_emit's .index offsets scan, the payload
// gather over gather_tiles 8 KB output tiles (past Ctl.out_data_len they return at once; no filter: Params.bloom.words is
// null), per-destination file offsets.
void launch_phase2(dbeel_engine *e, const Params &p, const uint4 *split, uint64_t n, uint64_t gather_tiles) {
    cudaStream_t s = e->stream;
    const uint32_t tiles = (uint32_t)((n + kResolveThreads - 1) / kResolveThreads);
    launch_k(e, k_scan_tile_sums, tiles, kResolveThreads, 0, s, p, split);
    launch_k(e, k_scan_tiles, (tiles + 1023) / 1024, 1024, 0, s, p);
    launch_k(e, k_scan_chunks, 1, 1024, 0, s, p);
    launch_k(e, k_emit, tiles, kResolveThreads, 0, s, p, split);
    launch_k(e, k_gather_h, (uint32_t)gather_tiles, kGhThreads, 0, s, p);
    launch_k(e, k_rebase_index, (uint32_t)((n + 255) / 256), 256, 0, s, p);
}

// Enqueued behind the kernels that wrote sp.flat / sp.dest (totals zeroed, the stop word set); sp, rp and p come from
// split_bind.  The split publishes to the mapped pinned block at pin_tot.  `sized(totals)` runs on them before the caps are
// checked: DBEEL_ERR_CAPACITY (nothing written, *items / *bytes = the required sizes) is the caller's to report.  Then
// phase 2 writes the output; ms_total runs from EV_START.
template <class F>
int split_emit(dbeel_engine *e, const SplitLayout &w, const ScanParams &sp, RouteParams rp, Params p, uint64_t pin_tot, bool device,
               dbeel_out *out, uint32_t *launches, uint64_t *items_out, uint64_t *bytes_out, F &&sized) {
    cudaStream_t s = e->stream;
    uint8_t *ws = e->ws, *h = e->pin;
    const uint32_t nd = w.nd;
    rp.n = w.n;
    rp.n_blocks = w.n_blocks;
    launch_split(e, sp, rp, reinterpret_cast<unsigned long long *>(e->pin_dev + pin_tot));
    *launches += 4;
    unsigned long long *host_tot = reinterpret_cast<unsigned long long *>(e->pin + pin_tot);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));
    sized(static_cast<const unsigned long long *>(host_tot));
    uint64_t items = 0, bytes = 0;
    for (uint32_t d = 0; d < nd; d++) {
        items += host_tot[d];
        bytes += host_tot[nd + d];
    }
    *items_out = items;
    *bytes_out = bytes;
    if (bytes > out->data_cap || 16 * items > out->index_cap) return DBEEL_ERR_CAPACITY;
    if (device && ((bytes && !out->data) || (items && !out->index))) return fail(e, DBEEL_ERR_INVALID_ARG, "null output buffer");
    // What depends on the output size is sized now that it is known -- records that share .data bytes can make the output
    // larger than the inputs: the gather's tile_first (one entry per 8 KB output tile) and, for host callers, the staged
    // outputs.  They live in stage_out, so the phase-1 workspace (the split records) stays where it is.
    const uint64_t gather_tiles = (bytes + kGatherTileBytes - 1) / kGatherTileBytes;
    const uint64_t tf_bytes = align_up(4ull * (gather_tiles + 2), kAlign);
    int rc = ensure_device(e, &e->stage_out, &e->stage_out_cap,
                           tf_bytes + (device ? 0 : align_up(bytes + 16, kAlign) + align_up(16 * items + 16, kAlign)));
    if (rc) return rc;
    uint32_t *tile_first = reinterpret_cast<uint32_t *>(e->stage_out);
    uint8_t *o_data = device ? static_cast<uint8_t *>(out->data) : e->stage_out + tf_bytes;
    uint8_t *o_index = device ? static_cast<uint8_t *>(out->index) : e->stage_out + tf_bytes + align_up(bytes + 16, kAlign);

    // ---- phase 2: .index (k_emit's offsets scan), payload gather, per-destination file offsets
    if (items) {
        Ctl *hc = reinterpret_cast<Ctl *>(h);
        memset(hc, 0, sizeof(Ctl));
        hc->span = (uint32_t)items;
        hc->total = (uint32_t)items;
        unsigned long long *hm = reinterpret_cast<unsigned long long *>(h + (w.o_memtab - w.o_ctl));
        unsigned long long before_b = 0, before_i = 0;
        for (uint32_t d = 0; d <= nd; d++) {
            hm[2 * d] = before_b;
            hm[2 * d + 1] = before_i;
            if (d < nd) { before_b += host_tot[nd + d]; before_i += host_tot[d]; }
        }
        p.tile_first = tile_first;
        p.tile_first_n = (uint32_t)(gather_tiles + 2);
        p.data_bound = bytes;
        p.out_data = o_data;
        p.out_index = reinterpret_cast<uint4 *>(o_index);
        launch_k(e, k_copy_words, (uint32_t)((w.header2_bytes / 4 + 255) / 256), 256, 0, s, reinterpret_cast<uint32_t *>(ws + w.o_ctl),
                 reinterpret_cast<const uint32_t *>(e->pin_dev), (uint32_t)(w.header2_bytes / 4));
        launch_phase2(e, p, rp.out_index, items, gather_tiles);
        *launches += 7;
    }
    CU(cudaEventRecord(e->ev[EV_GATHER], s));
    CU(cudaGetLastError());
    if (!device) {
        if (bytes) CU(cudaMemcpyAsync(out->data, o_data, bytes, cudaMemcpyDeviceToHost, s));
        if (items) CU(cudaMemcpyAsync(out->index, o_index, 16 * items, cudaMemcpyDeviceToHost, s));
    }
    CU(cudaStreamSynchronize(s));
    cudaEventElapsedTime(&e->stats.ms_total, e->ev[EV_START], e->ev[EV_GATHER]);
    e->stats.kernel_launches = *launches;
    e->stats.entries_out = items;
    e->stats.output_bytes = bytes + 16 * items;
    e->stats.gather_bytes = 2 * bytes + 16 * items + 8 * items;
    out->data_len = bytes;
    out->index_len = 16 * items;
    out->items_written = items;
    return DBEEL_OK;
}

int scan_entry(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges, uint32_t n_ranges,
               dbeel_out *out, dbeel_job_result *results, dbeel_scan_stop *stop, bool device) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    uint64_t key_bytes = 0;
    if (const int arc = scan_args(e, tables, n_tables, kind, ranges, n_ranges, results, stop, &key_bytes)) return arc;
    const Claim c(e);
    if (c.rc) return c.rc;
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    clear_scan(results, n_ranges, stop);
    uint64_t n64 = 0, data_total = 0, index_total = 0;
    unsigned long long stop0 = ~0ull; // an empty table: its first index read runs past EOF
    for (uint32_t t = 0; t < n_tables; t++) {
        const dbeel_table &tb = tables[t];
        if ((tb.data_len && !tb.data) || (tb.index_len >= 16 && !tb.index)) return fail(e, DBEEL_ERR_INVALID_ARG, "null table buffer");
        if (device && ((uintptr_t)tb.index & 15)) return fail(e, DBEEL_ERR_INVALID_ARG, "device .index buffers must be 16-byte aligned");
        if (tb.index_len < 16 && stop0 == ~0ull) stop0 = (n64 << 12) | ((unsigned long long)t << 2) | kScanStopPanic;
        n64 += tb.index_len / DBEEL_INDEX_ENTRY_SIZE;
        data_total += tb.data_len;
        index_total += tb.index_len;
    }
    if (n64 >= 0xFFFFFFF0ull) return fail(e, DBEEL_ERR_INVALID_ARG, "too many index records");
    if (device && (((uintptr_t)out->data | (uintptr_t)out->index) & 15))
        return fail(e, DBEEL_ERR_INVALID_ARG, "device output buffers must be 16-byte aligned");
    e->stats.input_bytes = data_total + index_total;
    e->stats.entries_in = n64;
    const uint32_t n = (uint32_t)n64;
    std::vector<uint32_t> base(n_tables + 1, 0);
    for (uint32_t t = 0; t < n_tables; t++) base[t + 1] = base[t] + (uint32_t)(tables[t].index_len / DBEEL_INDEX_ENTRY_SIZE);
    auto set_stop = [&](unsigned long long key) {
        if (key == ~0ull) return;
        const uint32_t t = (uint32_t)((key >> 2) & 1023);
        *stop = dbeel_scan_stop{(int32_t)t, (uint32_t)(key & 3), (key >> 12) - base[t]};
    };
    if (n == 0) { set_stop(stop0); return DBEEL_OK; }
    cudaStream_t s = e->stream;

    // host tables go down whole
    std::vector<ScanTable> td(n_tables);
    if (!device) {
        std::vector<HostPiece> pieces;
        for (uint32_t t = 0; t < n_tables; t++)
            pieces.insert(pieces.end(), {{tables[t].data, tables[t].data_len, nullptr}, {tables[t].index, tables[t].index_len, nullptr}});
        if (const int rc = stage_host(e, pieces)) return rc;
        for (uint32_t t = 0; t < n_tables; t++)
            td[t] = ScanTable{pieces[2 * t].dev, tables[t].data_len, reinterpret_cast<const uint4 *>(pieces[2 * t + 1].dev), base[t + 1] - base[t], base[t]};
    } else {
        for (uint32_t t = 0; t < n_tables; t++)
            td[t] = ScanTable{static_cast<const uint8_t *>(tables[t].data), tables[t].data_len, static_cast<const uint4 *>(tables[t].index),
                              base[t + 1] - base[t], base[t]};
    }

    // ---- workspace (the engine's grow-only one: a compaction after a scan reuses it as it is)
    const uint32_t nd = n_ranges;
    uint64_t off = 0;
    // header block, one copy through the mapped pinned block: tables | hash ranges or key offsets | range keys
    const uint64_t o_tab = carve_ws(&off, sizeof(ScanTable) * n_tables);
    const RangeHeader rh = carve_ranges(&off, kind, nd, key_bytes);
    const SplitLayout w = carve_split(&off, n, nd);
    int rc = ensure_device(e, &e->ws, &e->ws_cap, off);
    const uint64_t pin_tot = align_up(std::max(rh.bytes, w.header2_bytes), 64);
    if (!rc) rc = ensure_pinned(e, pin_tot + 8ull * (3 * nd + 1));
    if (rc) return rc;
    uint8_t *ws = e->ws;
    memcpy(e->pin + o_tab, td.data(), sizeof(ScanTable) * n_tables);

    ScanParams sp = {};
    RouteParams rp;
    Params p;
    sp.tables = reinterpret_cast<const ScanTable *>(ws + o_tab);
    sp.n_tables = n_tables;
    sp.n = n;
    split_bind(w, ws, &sp, &rp, &p);
    sp.stop0 = stop0;

    // ---- phase 1: classify; the split and phase 2 (split_emit) size the output from what it selected
    uint32_t launches = 0;
    CU(cudaEventRecord(e->ev[EV_START], s));
    land_ranges(e, rh, kind, ranges, nd, key_bytes, &sp);
    CU(cudaMemsetAsync(ws + w.o_tot, 0, 8ull * 3 * nd, s));
    CU(cudaMemsetAsync(sp.stop, 0xFF, 8, s));
    launch_k(e, k_scan_classify, (n + 255) / 256, 256, 0, s, sp);
    launches += 2;
    uint64_t items = 0, bytes = 0;
    rc = split_emit(e, w, sp, rp, p, pin_tot, device, out, &launches, &items, &bytes, [&](const unsigned long long *host_tot) {
        const unsigned long long stop_key = std::min<unsigned long long>(host_tot[3 * nd], stop0);
        set_stop(stop_key);
        e->stats.entries_valid = stop_key == ~0ull ? n : (stop_key >> 12);
        uint64_t it = 0, by = 0;
        for (uint32_t d = 0; d < nd; d++) {
            dbeel_job_result &r = results[d];
            r.data_off = by;
            r.data_len = host_tot[nd + d];
            r.index_off = 16 * it;
            r.items_written = host_tot[d];
            r.index_len = 16 * host_tot[d];
            it += host_tot[d];
            by += host_tot[nd + d];
        }
    });
    if (rc == DBEEL_ERR_CAPACITY) {
        std::fill_n(results, nd, dbeel_job_result{});
        return fail(e, DBEEL_ERR_CAPACITY, "scan output larger than the buffers (index records that overlap in .data)");
    }
    return rc;
}


// ------------------------------------------------------------------------------------ N2 with values: dbeel_get_values*
// k_lookup_emit writes the rows and, per query, its hit's entry as a split record for destination 0 (or kScanNone: no
// entry); split_emit turns those into one arrival batch in query order.  Only the rows and the selected bytes come back.
int get_values_entry(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys, const uint64_t *key_off,
                     uint64_t n_keys, uint32_t mode, dbeel_out *out, dbeel_lookup_result *results, bool device) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (const int arc = lookup_args(e, tables, n_tables, key_off, n_keys, mode, results)) return arc;
    if (n_keys >= 0xFFFFFFF0ull) return fail(e, DBEEL_ERR_INVALID_ARG, "2^32 - 16 keys or more");
    if (device && (((uintptr_t)out->data | (uintptr_t)out->index) & 15))
        return fail(e, DBEEL_ERR_INVALID_ARG, "device output buffers must be 16-byte aligned");
    const Claim c(e);
    if (c.rc) return c.rc;
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    if (n_keys == 0) return DBEEL_OK;
    cudaStream_t s = e->stream;
    const uint32_t n = (uint32_t)n_keys;
    uint64_t off = 0;
    const uint64_t o_desc = carve_ws(&off, sizeof(TableDesc) * n_tables);
    const uint64_t o_rows = carve_ws(&off, device ? 0 : 16ull * n); // host callers: the rows before their D2H
    const SplitLayout w = carve_split(&off, n, 1);
    int rc = ensure_device(e, &e->ws, &e->ws_cap, off);
    if (rc) return rc;
    const uint64_t pin_tot = align_up(w.header2_bytes, 64);
    const uint8_t *d_keys;
    const uint64_t *d_off;
    rc = stage_lookup(e, tables, n_tables, keys, key_off, n_keys, device, pin_tot + 8ull * 4, reinterpret_cast<TableDesc *>(e->ws + o_desc),
                      &d_keys, &d_off);
    if (rc) return rc;
    uint8_t *ws = e->ws;
    ScanParams sp = {};
    RouteParams rp;
    Params p;
    split_bind(w, ws, &sp, &rp, &p);
    uint4 *d_res = device ? reinterpret_cast<uint4 *>(results) : reinterpret_cast<uint4 *>(ws + o_rows);
    LookupParams lp{reinterpret_cast<const TableDesc *>(ws + o_desc), n_tables, mode, d_keys, d_off, n_keys, d_res};
    e->stats.entries_in = n_keys;
    uint32_t launches = 1;
    CU(cudaEventRecord(e->ev[EV_START], s));
    CU(cudaMemsetAsync(ws + w.o_tot, 0, 8ull * 3, s));
    CU(cudaMemsetAsync(sp.stop, 0xFF, 8, s));
    launch_k(e, k_lookup_emit, (n + 255) / 256, 256, 0, s, lp, LookupEmit{sp.dest, sp.flat});
    if (!device) CU(cudaMemcpyAsync(results, d_res, 16ull * n, cudaMemcpyDeviceToHost, s)); // back with the sizes: filled on ERR_CAPACITY too
    uint64_t items = 0, bytes = 0;
    rc = split_emit(e, w, sp, rp, p, pin_tot, device, out, &launches, &items, &bytes, [](const unsigned long long *) {});
    if (rc == DBEEL_ERR_CAPACITY) {
        out->data_len = bytes;
        out->index_len = 16 * items;
        return fail(e, DBEEL_ERR_CAPACITY, "the entries found are larger than the output buffers (data_len / index_len: the sizes needed)");
    }
    return rc;
}


// ------------------------------------------------------------------------------------ N2 streamed: dbeel_get_values_stream
// Ranges of one file laid out in a staging buffer: run k (merged ranges) at pos[k], congruent to its file offset modulo 16
// with 16 bytes of slack on both sides, so the kernels' aligned 8-byte loads stay inside the buffer.
struct GvsStaged {
    std::vector<ByteRange> runs;
    std::vector<uint64_t> pos;
    uint64_t end = 0;
    uint64_t at(uint64_t off) const { // staging position of file offset `off` (inside some run)
        const size_t k = std::upper_bound(runs.begin(), runs.end(), off, [](uint64_t o, const ByteRange &r) { return o < r.lo; }) - runs.begin() - 1;
        return pos[k] + (off - runs[k].lo);
    }
};

GvsStaged gvs_stage(std::vector<ByteRange> r, uint64_t gap, uint64_t base) {
    GvsStaged s;
    s.runs = merge_ranges(std::move(r), gap);
    uint64_t p = base;
    for (const ByteRange &x : s.runs) {
        const uint64_t at = align_up(p + 16, 16) + (x.lo & 15);
        s.pos.push_back(at);
        p = at + (x.hi - x.lo) + 16;
    }
    s.end = align_up(p, kAlign);
    return s;
}

// Every run of `s` of table t's file `kind` into dst + pos, through the read callback from a few threads, in pieces of at
// most StreamPump::kPiece bytes; the callback's code comes back unchanged.  A batch of many small reads (fences, scattered
// hits) is dominated by the per-call cost, so this takes parallel_pieces' lock-free loop rather than the pump's
// partition-ordered one.
int gvs_read(dbeel_engine *e, const dbeel_scan_io *io, uint32_t t, uint32_t kind, const GvsStaged &s, uint8_t *dst) {
    struct Piece { uint64_t off, len; uint8_t *dst; };
    std::vector<Piece> ps;
    for (size_t k = 0; k < s.runs.size(); k++) {
        const uint64_t len = s.runs[k].hi - s.runs[k].lo;
        for (uint64_t done = 0; done < len; done += StreamPump::kPiece)
            ps.push_back({s.runs[k].lo + done, std::min(len - done, StreamPump::kPiece), dst + s.pos[k] + done});
        e->stats.input_bytes += len;
    }
    return parallel_pieces(ps.size(), [&](size_t k) { return io->read(io->ctx, t, kind, ps[k].off, ps[k].len, ps[k].dst); });
}

// The fences of the open internal nodes of pt, through the callback: their index records (runs closer than
// kLookupMergeGap as one read) into fix[k], then their key frames of up to max_klen key bytes (runs that touch as one
// read) into frames, staged by sf.  has[k]: node k's record points inside .data and its frame is frame[k].
struct GvsFenceReads {
    std::vector<uint4> fix;
    std::vector<ByteRange> frame;
    std::vector<uint8_t> has;
    GvsStaged sf;
    std::vector<uint8_t> frames;
    uint64_t image_bytes() const { return 24 * fix.size() + sf.end; } // gvs_fence_image
};

int gvs_read_fences(dbeel_engine *e, const dbeel_scan_io *io, uint32_t ti, const ProbeTree &pt, uint64_t data_len, uint64_t max_klen,
                    GvsFenceReads *f) {
    const uint32_t mode = pt.mode;
    const uint64_t leaf0 = 1ull << pt.depth;
    int rc;
    std::vector<ByteRange> ir;
    for (uint64_t k = 1; k < leaf0; k++)
        if (pt.open[k]) { const uint64_t p = search_pos(mode, pt.state[k]); ir.push_back({16 * p, 16 * p + 16}); }
    const GvsStaged si = gvs_stage(ir, kLookupMergeGap, 0);
    if ((rc = ensure_host(e, &e->ring_out, &e->ring_out_cap, si.end))) return rc;
    if ((rc = gvs_read(e, io, ti, DBEEL_STREAM_INDEX, si, e->ring_out))) return fail(e, rc, "stream read callback failed (.index, fences)");
    f->fix.assign(leaf0, make_uint4(0, 0, 0, 0));
    f->has.assign(leaf0, 0);
    f->frame.assign(leaf0, ByteRange{0, 0});
    std::vector<ByteRange> fr;
    for (uint64_t k = 1; k < leaf0; k++) {
        if (!pt.open[k]) continue;
        memcpy(&f->fix[k], e->ring_out + si.at(16 * search_pos(mode, pt.state[k])), 16);
        if (probe_frame(reinterpret_cast<const uint8_t *>(&f->fix[k]), data_len, max_klen, &f->frame[k])) { f->has[k] = 1; fr.push_back(f->frame[k]); }
    }
    f->sf = gvs_stage(fr, 0, 0);
    f->frames.resize(f->sf.end);
    if ((rc = gvs_read(e, io, ti, DBEEL_STREAM_DATA, f->sf, f->frames.data()))) return fail(e, rc, "stream read callback failed (.data, fences)");
    return DBEEL_OK;
}

// node k's frame address: its staged frame at `frame` (host view `host`), or 0 when its length prefix runs past .data
// (as probe(): the record is reported corrupt)
inline unsigned long long gvs_frame_addr(const GvsFenceReads &f, uint64_t k, uint64_t data_len, const uint8_t *host, const uint8_t *dev) {
    if (!f.has[k] || rd64(host) > data_len - f.frame[k].lo - 8) return 0;
    return reinterpret_cast<unsigned long long>(dev);
}

// The fences of one table read for one call, as GvsFences descends them: fix[2^depth] | ffr[2^depth] | frames, written
// at img (host, image_bytes()) for a device copy at dev, which ffr points into.  With dev 16-aligned and depth >= 1, every
// frame stays congruent to its file offset modulo 16.
void gvs_fence_image(const GvsFenceReads &f, uint64_t data_len, uint8_t *img, uint8_t *dev) {
    const uint64_t leaf0 = f.fix.size(), o_frames = 24 * leaf0;
    memcpy(img, f.fix.data(), 16 * leaf0);
    memcpy(img + o_frames, f.frames.data(), f.sf.end);
    unsigned long long *ffr = reinterpret_cast<unsigned long long *>(img + 16 * leaf0);
    for (uint64_t k = 0; k < leaf0; k++) {
        const uint64_t p = o_frames + (f.has[k] ? f.sf.at(f.frame[k].lo) : 0);
        ffr[k] = gvs_frame_addr(f, k, data_len, img + p, dev + p);
    }
}

} // namespace

// ---- readers (dbeel_reader_*): what dbeel_get_values_stream would read again on every call, kept on the device
// One table of a reader (a tree shares it between its readers): the filter, uploaded when the table is created, and per
// mode the fences of the top `depth` levels (host/lookup_plan.h), read the first time a batch in that mode reaches it.
struct dbeel_reader_table {
    int device = 0;
    uint64_t id = next_id(); // the page cache's key for the table's files: process-wide, never reused
    TableDesc desc = {};      // data / index unset; words -> the resident filter, or nullptr
    uint8_t *bloom_dev = nullptr;
    int32_t depth = -1;       // D_t: chosen by the first reader that includes the table, kept after
    struct Fences {
        bool loaded = false;
        ProbeTree pt;         // the leaves' intervals (the node states of the cached levels)
        uint8_t *dev = nullptr; // fix[2^depth] | ffr[2^depth] | frame slots (kReaderFrameSlot bytes per node)
    } fences[2];
    ~dbeel_reader_table() {
        cudaSetDevice(device);
        if (bloom_dev) cudaFree(bloom_dev);
        for (auto &f : fences)
            if (f.dev) cudaFree(f.dev);
    }
    static uint64_t next_id() {
        static std::atomic<uint64_t> n{1};
        return n.fetch_add(1);
    }
};

struct dbeel_reader {
    dbeel_engine *e = nullptr;
    std::vector<ReaderTableRef> tables;
    dbeel_scan_io io = {};
    std::shared_ptr<void> owner; // what io.ctx points at, when the reader owns it (tree readers)
    dbeel_page_cache *cache = nullptr; // dbeel_reader_attach_page_cache
};

// The readers' page cache: its slots in one device allocation, the page table and CLOCK on the host (host/page_cache.h).
struct dbeel_page_cache {
    dbeel_engine *e = nullptr;
    uint8_t *pool = nullptr; // pc.capacity() slots of kPageBytes
    PageCache pc;
    uint8_t *host = nullptr; // page-locked staging of one request: its miss image, then its copy list (grow-only)
    uint64_t host_cap = 0;
    explicit dbeel_page_cache(uint64_t slots) : pc(slots) {}
    ~dbeel_page_cache() {
        if (pool) cudaFree(pool);
        if (host) cudaFreeHost(host);
    }
};

namespace {

// Reads the fences of reader table rt (table ti of the batch) in `mode` at its depth, into its own device block.  The
// frames hold at most kReaderFrameCap key bytes.  The host image goes down from ring_out, which the leaf groups refill
// only after the touched read-back has synchronised the stream.
int reader_load_fences(dbeel_engine *e, const dbeel_scan_io *io, uint32_t ti, dbeel_reader_table *rt, uint32_t mode) {
    dbeel_reader_table::Fences &c = rt->fences[mode];
    plan_probe_tree(mode, rt->desc.n, (uint32_t)rt->depth, &c.pt);
    const uint64_t leaf0 = 1ull << rt->depth, data_len = rt->desc.data_len;
    if (rt->depth > 0) {
        GvsFenceReads fr;
        int rc = gvs_read_fences(e, io, ti, c.pt, data_len, kReaderFrameCap, &fr);
        if (rc) return rc;
        const uint64_t o_ffr = 16 * leaf0, o_slot = o_ffr + 8 * leaf0, bytes = o_slot + kReaderFrameSlot * leaf0;
        if ((rc = ensure_host(e, &e->ring_out, &e->ring_out_cap, bytes))) return rc;
        if (c.dev) cudaFree(c.dev); // a load whose copy failed
        if (cudaMalloc(reinterpret_cast<void **>(&c.dev), bytes) != cudaSuccess) {
            cudaGetLastError();
            c.dev = nullptr;
            return fail(e, DBEEL_ERR_NOMEM, "cudaMalloc(reader fences)");
        }
        uint8_t *img = e->ring_out;
        memset(img + o_slot, 0, kReaderFrameSlot * leaf0);
        memcpy(img, fr.fix.data(), 16 * leaf0);
        unsigned long long *ffr = reinterpret_cast<unsigned long long *>(img + o_ffr);
        for (uint64_t k = 0; k < leaf0; k++) {
            uint8_t *slot = img + o_slot + kReaderFrameSlot * k;
            if (fr.has[k]) memcpy(slot, fr.frames.data() + fr.sf.at(fr.frame[k].lo), fr.frame[k].hi - fr.frame[k].lo);
            ffr[k] = gvs_frame_addr(fr, k, data_len, slot, c.dev + o_slot + kReaderFrameSlot * k);
        }
        CU(cudaMemcpyAsync(c.dev, img, bytes, cudaMemcpyHostToDevice, e->stream));
    }
    c.loaded = true;
    return DBEEL_OK;
}

// One staged image of file `kind`: the runs of every part's GvsStaged (table t of the batch) at their positions, which lie
// in [from, to) of `host` (page-locked) and `dev`.  Without a page cache, or when the request needs more pages than the
// cache has slots, that is gvs_read into host and one H2D of [from, to).  With a cache attached to reader r, the pages it
// holds are copied on the device, and the missing ones are read through the callback into the cache's staging (page-aligned
// runs clipped to the file's length, host/page_cache.h), go down with the copy list to stage_out, and one k_page_copy fills
// their slots and the image from them; host_too brings the image back to host (the .index slices, whose records the host
// reads).  The pages become resident only once their reads have succeeded.  The caller has synchronised the stream since
// its last use of stage_out and of the cache's staging.  The callback's code comes back unchanged, with `what`.
struct GvsPart {
    uint32_t t; // the table's position in its reader's (or the call's) tables: the callback's table argument
    const GvsStaged *s;
    const dbeel_reader *r = nullptr;
    const dbeel_scan_io *io = nullptr;
};

int gvs_load(dbeel_engine *e, uint32_t kind, const std::vector<GvsPart> &parts, uint8_t *host, uint8_t *dev, uint64_t from,
             uint64_t to, bool host_too, const char *what) {
    cudaStream_t s = e->stream;
    int rc;
    // the parts of each page cache, in order of first appearance, as one request each
    std::vector<dbeel_page_cache *> cs;
    std::vector<std::vector<size_t>> of;
    std::vector<PagePlan> plans;
    for (size_t k = 0; k < parts.size(); k++) {
        dbeel_page_cache *c = parts[k].r ? parts[k].r->cache : nullptr;
        if (!c) continue;
        const size_t ci = std::find(cs.begin(), cs.end(), c) - cs.begin();
        if (ci == cs.size()) { cs.push_back(c); of.emplace_back(); }
        of[ci].push_back(k);
    }
    std::vector<uint8_t> direct(parts.size(), 1);
    uint64_t stage_bytes = 0;
    for (size_t ci = 0; ci < cs.size(); ci++) {
        std::vector<PagePart> pp;
        for (size_t k : of[ci]) {
            const GvsPart &g = parts[k];
            const TableDesc &d = g.r->tables[g.t]->desc;
            pp.push_back(PagePart{g.r->tables[g.t]->id, kind, kind == DBEEL_STREAM_DATA ? d.data_len : 16 * d.n, {}});
            for (size_t j = 0; j < g.s->runs.size(); j++) pp.back().ranges.push_back(PageRange{g.s->runs[j].lo, g.s->runs[j].hi, g.s->pos[j]});
        }
        plans.push_back(cs[ci]->pc.plan(pp, StreamPump::kPiece));
        const PagePlan &p = plans.back();
        if (p.bypass) continue;
        for (size_t k : of[ci]) direct[k] = 0;
        stage_bytes = std::max(stage_bytes, align_up(p.img_bytes, kAlign) + sizeof(PageCopy) * p.moves.size());
    }
    auto drop = [&](size_t from_ci) { // plans not carried out leave their caches as they were
        for (size_t ci = from_ci; ci < cs.size(); ci++)
            if (!plans[ci].bypass) cs[ci]->pc.commit(plans[ci], false);
    };
    rc = stage_bytes ? ensure_device(e, &e->stage_out, &e->stage_out_cap, std::max<uint64_t>(stage_bytes, 256)) : DBEEL_OK;
    if (rc) { drop(0); return rc; }
    // uncached parts (no cache, or a request larger than its cache): read into host, the whole image down in one copy,
    // before any page copy writes its own parts over it
    bool any_direct = false, any_paged = false;
    for (size_t k = 0; k < parts.size(); k++) {
        if (!direct[k]) { any_paged = true; continue; }
        any_direct = true;
        if ((rc = gvs_read(e, parts[k].io, parts[k].t, kind, *parts[k].s, host))) { drop(0); return fail(e, rc, what); }
    }
    if (any_direct && to > from) {
        const cudaError_t ce = cudaMemcpyAsync(dev + from, host + from, to - from, cudaMemcpyHostToDevice, s);
        if (ce != cudaSuccess) { drop(0); return fail(e, DBEEL_ERR_CUDA, "cudaMemcpyAsync", ce); }
    }
    for (size_t ci = 0; ci < cs.size(); ci++) {
        dbeel_page_cache *c = cs[ci];
        PagePlan &p = plans[ci];
        if (p.bypass) continue;
        const uint64_t o_copy = align_up(p.img_bytes, kAlign), bytes = o_copy + sizeof(PageCopy) * p.moves.size();
        rc = ensure_host(e, &c->host, &c->host_cap, std::max<uint64_t>(bytes, 256));
        if (rc) { drop(ci); return rc; }
        for (const PageRead &x : p.reads) e->stats.input_bytes += x.len;
        rc = parallel_pieces(p.reads.size(), [&](size_t k) {
            const PageRead &x = p.reads[k];
            const GvsPart &g = parts[of[ci][x.part]];
            return g.io->read(g.io->ctx, g.t, kind, x.off, x.len, c->host + x.img);
        });
        if (rc) { drop(ci); return fail(e, rc, what); }
        const uint64_t src[3] = {(uint64_t)e->stage_out, (uint64_t)e->stage_out, (uint64_t)c->pool}; // by PageMove::how
        const uint64_t dst[3] = {(uint64_t)c->pool, (uint64_t)dev, (uint64_t)dev};
        PageCopy *pc = reinterpret_cast<PageCopy *>(c->host + o_copy);
        for (size_t k = 0; k < p.moves.size(); k++) {
            const PageMove &m = p.moves[k];
            pc[k] = PageCopy{src[m.how] + m.src, dst[m.how] + m.dst, m.len, 0};
        }
        cudaError_t ce = cudaSuccess;
        if (!p.moves.empty()) {
            ce = cudaMemcpyAsync(e->stage_out, c->host, bytes, cudaMemcpyHostToDevice, s);
            if (ce == cudaSuccess) {
                launch_k(e, k_page_copy, (uint32_t)((32 * p.moves.size() + 255) / 256), 256, 0, s, reinterpret_cast<const PageCopy *>(e->stage_out + o_copy),
                         (uint64_t)p.moves.size());
                ce = cudaGetLastError();
            }
        }
        c->pc.commit(p, ce == cudaSuccess); // the copies that read a slot are enqueued before any later fill of it
        if (ce != cudaSuccess) { drop(ci + 1); return fail(e, DBEEL_ERR_CUDA, "k_page_copy", ce); }
    }
    if (any_paged && host_too && to > from) {
        CU(cudaMemcpyAsync(host + from, dev + from, to - from, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
    }
    return DBEEL_OK;
}

// Where the touched leaves of part t of a group come from: the reader (null: none) and io its reads go through, the table's
// position there, its .data length and the longest key of the batch that searches it.
struct LeafSrc {
    const dbeel_reader *r;
    const dbeel_scan_io *io;
    uint32_t table;
    uint64_t data_len, max_klen;
};

// One group of touched leaves (group_leaves), ascending (part, leaf), on the device for k_lookup_leaf: per
// part its index slices into stage_in behind the header (through ring_in, and back to it), then the .data windows of
// those slices (leaf_window) into stage_in2 (through ring_out).  The header at stage_in is GvsLeaf[nl] | first[nt + 1]
// (nt = src.size()): part t's leaves are [first[t], first[t + 1]), each biased so that record r of the table lies
// at index + r and file offset o at data + o (a leaf whose records all point past the file never dereferences data:
// probe() reports them corrupt first).  Through gvs_load, so with a page cache this also writes stage_out.
int gvs_load_leaves(dbeel_engine *e, const std::vector<LeafSrc> &src, const TouchedLeaf *lv, uint32_t nl) {
    const uint32_t nt = (uint32_t)src.size();
    std::vector<uint32_t> first(nt + 1, 0);
    for (uint32_t k = 0; k < nl; k++) first[lv[k].t + 1]++;
    for (uint32_t t = 0; t < nt; t++) first[t + 1] += first[t];
    const uint64_t o_first = sizeof(GvsLeaf) * nl, hdr = align_up(o_first + 4ull * (nt + 1), kAlign);
    std::vector<GvsStaged> ss(nt), sw(nt);
    std::vector<GvsPart> parts;
    uint64_t end = hdr;
    for (uint32_t t = 0; t < nt; t++) {
        if (first[t] == first[t + 1]) continue;
        std::vector<ByteRange> x;
        for (uint32_t k = first[t]; k < first[t + 1]; k++) x.push_back({16 * lv[k].a, 16 * lv[k].b});
        ss[t] = gvs_stage(std::move(x), kLookupMergeGap, end);
        end = ss[t].end;
        parts.push_back(GvsPart{src[t].table, &ss[t], src[t].r, src[t].io});
    }
    int rc = ensure_host(e, &e->ring_in, &e->ring_in_cap, end);
    if (!rc) rc = ensure_device(e, &e->stage_in, &e->stage_in_cap, end);
    if (rc) return rc;
    if ((rc = gvs_load(e, DBEEL_STREAM_INDEX, parts, e->ring_in, e->stage_in, hdr, end, true, "stream read callback failed (.index, leaves)")))
        return rc;
    std::vector<ByteRange> win(nl);
    std::vector<uint8_t> has(nl, 0);
    uint64_t wend = 0;
    parts.clear();
    for (uint32_t t = 0; t < nt; t++) {
        if (first[t] == first[t + 1]) continue;
        std::vector<ByteRange> wr;
        for (uint32_t k = first[t]; k < first[t + 1]; k++)
            if (leaf_window(e->ring_in + ss[t].at(16 * lv[k].a), lv[k].b - lv[k].a, src[t].data_len, src[t].max_klen, &win[k])) {
                has[k] = 1;
                wr.push_back(win[k]);
            }
        sw[t] = gvs_stage(std::move(wr), 0, wend);
        wend = sw[t].end;
        if (!sw[t].runs.empty()) parts.push_back(GvsPart{src[t].table, &sw[t], src[t].r, src[t].io});
    }
    rc = ensure_host(e, &e->ring_out, &e->ring_out_cap, std::max<uint64_t>(wend, 256));
    if (!rc) rc = ensure_device(e, &e->stage_in2, &e->stage_in2_cap, std::max<uint64_t>(wend, 256));
    if (rc) return rc;
    if ((rc = gvs_load(e, DBEEL_STREAM_DATA, parts, e->ring_out, e->stage_in2, 0, wend, false, "stream read callback failed (.data, leaves)")))
        return rc;
    GvsLeaf *hl = reinterpret_cast<GvsLeaf *>(e->ring_in);
    for (uint32_t k = 0; k < nl; k++) {
        const uint32_t t = lv[k].t;
        const uint64_t lo = 16 * lv[k].a;
        const uintptr_t ib = reinterpret_cast<uintptr_t>(e->stage_in + ss[t].at(lo)) - lo;
        const uintptr_t db = has[k] ? reinterpret_cast<uintptr_t>(e->stage_in2 + sw[t].at(win[k].lo)) - win[k].lo
                                    : reinterpret_cast<uintptr_t>(e->stage_in2);
        hl[k] = GvsLeaf{reinterpret_cast<const uint8_t *>(db), reinterpret_cast<const uint4 *>(ib), lv[k].leaf, 0, 0};
    }
    memcpy(e->ring_in + o_first, first.data(), 4ull * (nt + 1));
    CU(cudaMemcpyAsync(e->stage_in, e->ring_in, hdr, cudaMemcpyHostToDevice, e->stream));
    return DBEEL_OK;
}

// One batch of a batched read from files: dbeel_get_values_stream's (r null: its tables' filters staged here, reads
// through io) or a reader's (its resident filters and cached fences, reads through its io and page cache).
struct GvsBatch {
    dbeel_reader *r = nullptr;
    const dbeel_scan_io *io = nullptr;
    std::vector<TableDesc> td; // oldest first
    const uint8_t *keys = nullptr;
    const uint64_t *key_off = nullptr;
    uint64_t n_keys = 0, max_klen = 0;
    uint32_t mode = 0;
};

// The hit heap (stage_out2) holds every answered entry of a walk until split_emit gathers them; it grows to `need` bytes
// keeping the `keep` it holds.
int gvs_heap_reserve(dbeel_engine *e, uint64_t need, uint64_t keep) {
    if (need <= e->stage_out2_cap) return DBEEL_OK;
    uint8_t *old = e->stage_out2;
    const uint64_t old_cap = e->stage_out2_cap;
    e->stage_out2 = nullptr;
    e->stage_out2_cap = 0;
    int rc = ensure_device(e, &e->stage_out2, &e->stage_out2_cap, need);
    if (!rc && old && keep) CU(cudaMemcpyAsync(e->stage_out2, old, std::min(old_cap, keep), cudaMemcpyDeviceToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    if (old) cudaFree(old);
    return rc;
}

// What the levels of a walk share: its queries on the device, where a level's pairs and touched flags go (the pairs go
// down from e->pin + p_pairs, the touched flags come back to e->pin), the leaf kernel's heap counter and the hit heap.
struct GvsLevel {
    GvsQueries gq;
    uint32_t grid;
    GvsPair *d_pairs;
    uint8_t *d_touched;
    uint64_t p_pairs;
    unsigned long long *d_need, *d_cursor;
    uint64_t heap_bound = 0; // the heap bytes the copies so far may have used
    uint32_t launches = 0, groups = 0;
};

// One level of a walk, from its pairs with their open-query counts known to its last leaf group.  A live pair whose pts[p]
// the caller has set has its fences (depth, fix, ffr) chosen; the others choose here from count[p] open queries (0: the
// pair is dropped): the reader table's cached fences when they serve the queries (reader_uses_cache), else fences read
// for this call into one image in stage_in.  Then one k_lookup_fence, one read-back of the touched leaves, and the leaves
// in groups (group_leaves over pairs, each reader's page cache a cache of its own), each with one k_lookup_leaf and, when
// the group's hits need heap bytes, one k_gvs_copy that moves their entries out of the window before it is reused.
// src[p]: where pair p's leaves come from.  Every phase ends in a stream synchronise before its pinned buffers are refilled.
template <bool kSeek>
int gvs_level(dbeel_engine *e, GvsLevel &L, std::vector<GvsPair> &pairs, const std::vector<LeafSrc> &src, const std::vector<uint64_t> &count,
              std::vector<const ProbeTree *> &pts) {
    cudaStream_t s = e->stream;
    const uint64_t budget = e->partition_bytes;
    const uint32_t np = (uint32_t)pairs.size();
    int rc;
    // ---- fences: the index records of the open internal nodes, then their key frames (or the reader's copies)
    std::vector<ProbeTree> pt_call(np);
    std::vector<GvsFenceReads> frs(np);
    std::vector<uint64_t> img_at(np, ~0ull), touched_at(np);
    uint64_t img_bytes = 0, tbytes = 0;
    bool any = false, any_fence = false;
    for (uint32_t b = 0; b < np; b++) {
        const LeafSrc &S = src[b];
        GvsPair &P = pairs[b];
        if (!P.live) continue;
        if (!pts[b]) {
            const uint64_t m = count[b];
            if (m == 0) { // no query reaches the table: nothing of it is read
                P.live = 0;
                continue;
            }
            const uint32_t ti = P.table;
            dbeel_reader_table *rt = S.r ? S.r->tables[ti].get() : nullptr;
            dbeel_reader_table::Fences *cache = rt ? &rt->fences[P.mode] : nullptr;
            const uint32_t cd = rt ? (uint32_t)rt->depth : 0;
            uint32_t depth = lookup_depth(m, P.t.n, P.t.data_len, 8 + S.max_klen, budget);
            if (cache && reader_uses_cache(S.max_klen, depth, cd)) {
                depth = cd;
                if (!cache->loaded) {
                    if ((rc = reader_load_fences(e, S.io, ti, rt, P.mode))) return rc;
                    CU(cudaStreamSynchronize(s)); // its image goes down from ring_out, which the next pair refills
                }
                pts[b] = &cache->pt;
                P.fix = reinterpret_cast<const uint4 *>(cache->dev);
                P.ffr = reinterpret_cast<const unsigned long long *>(cache->dev + (16ull << cd));
            } else {
                plan_probe_tree(P.mode, P.t.n, depth, &pt_call[b]);
                pts[b] = &pt_call[b];
                if (depth > 0) {
                    if ((rc = gvs_read_fences(e, S.io, ti, pt_call[b], P.t.data_len, S.max_klen, &frs[b]))) return rc;
                    img_at[b] = align_up(img_bytes, kAlign);
                    img_bytes = img_at[b] + frs[b].image_bytes();
                }
            }
            P.depth = depth;
        }
        touched_at[b] = tbytes;
        P.touched = L.d_touched + tbytes;
        tbytes += 1ull << P.depth;
        any = true;
        any_fence = any_fence || P.depth > 0;
    }
    if (!any) return DBEEL_OK;
    if (img_bytes) {
        if ((rc = ensure_host(e, &e->ring_in, &e->ring_in_cap, img_bytes))) return rc;
        if ((rc = ensure_device(e, &e->stage_in, &e->stage_in_cap, img_bytes))) return rc;
        for (uint32_t b = 0; b < np; b++) {
            if (img_at[b] == ~0ull) continue;
            gvs_fence_image(frs[b], pairs[b].t.data_len, e->ring_in + img_at[b], e->stage_in + img_at[b]);
            pairs[b].fix = reinterpret_cast<const uint4 *>(e->stage_in + img_at[b]);
            pairs[b].ffr = reinterpret_cast<const unsigned long long *>(e->stage_in + img_at[b] + (16ull << pairs[b].depth));
        }
        CU(cudaMemcpyAsync(e->stage_in, e->ring_in, img_bytes, cudaMemcpyHostToDevice, s));
    }
    CU(cudaMemsetAsync(L.d_touched, 0, tbytes, s));
    for (uint32_t b = 0; b < np; b++)
        if (pairs[b].live && pairs[b].depth == 0) CU(cudaMemsetAsync(L.d_touched + touched_at[b], 1, 1, s));
    memcpy(e->pin + L.p_pairs, pairs.data(), sizeof(GvsPair) * np);
    CU(cudaMemcpyAsync(L.d_pairs, e->pin + L.p_pairs, sizeof(GvsPair) * np, cudaMemcpyHostToDevice, s));
    if (any_fence) {
        launch_k(e, k_lookup_fence<kSeek>, L.grid, 256, 0, s, L.gq, static_cast<const GvsPair *>(L.d_pairs));
        L.launches++;
    }
    CU(cudaMemcpyAsync(e->pin, L.d_touched, tbytes, cudaMemcpyDeviceToHost, s));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));

    // ---- leaves, in groups of about `budget` bytes (with page caches, each cache's leaves at most its capacity)
    std::vector<uint64_t> cache_bytes;
    std::vector<dbeel_page_cache *> caches;
    std::vector<TouchedLeaf> lv;
    std::vector<LeafPair> lp(np);
    for (uint32_t b = 0; b < np; b++) {
        const GvsPair &P = pairs[b];
        dbeel_page_cache *c = src[b].r ? src[b].r->cache : nullptr;
        int32_t ci = -1;
        if (c) {
            ci = (int32_t)(std::find(caches.begin(), caches.end(), c) - caches.begin());
            if (ci == (int32_t)caches.size()) {
                caches.push_back(c);
                cache_bytes.push_back(kPageBytes * c->pc.capacity());
            }
        }
        lp[b] = LeafPair{P.t.n, P.t.data_len, src[b].max_klen, ci};
        if (P.live) touched_leaves(*pts[b], b, e->pin + touched_at[b], &lv);
    }
    const std::vector<size_t> cut = group_leaves(lv, lp, budget, cache_bytes);
    for (size_t gi = 0; gi + 1 < cut.size(); gi++) {
        const uint32_t nl = (uint32_t)(cut[gi + 1] - cut[gi]);
        if ((rc = gvs_load_leaves(e, src, lv.data() + cut[gi], nl))) return rc;
        CU(cudaMemsetAsync(L.d_need, 0, 8, s));
        launch_k(e, k_lookup_leaf<kSeek>, L.grid, 256, 0, s, L.gq, static_cast<const GvsPair *>(L.d_pairs),
                 reinterpret_cast<const GvsLeaf *>(e->stage_in), reinterpret_cast<const uint32_t *>(e->stage_in + sizeof(GvsLeaf) * nl), L.d_need);
        CU(cudaMemcpyAsync(e->pin, L.d_need, 8, cudaMemcpyDeviceToHost, s));
        CU(cudaGetLastError());
        CU(cudaStreamSynchronize(s));
        L.launches++;
        if (const uint64_t need = rd64(e->pin)) { // the group's hits leave the window for the heap before it is reused
            if ((rc = gvs_heap_reserve(e, L.heap_bound + need, L.heap_bound))) return rc;
            L.heap_bound += need;
            launch_k(e, k_gvs_copy, (uint32_t)((32 * L.gq.n_keys + 255) / 256), 256, 0, s, L.gq, e->stage_out2, L.d_cursor);
            CU(cudaGetLastError());
            CU(cudaStreamSynchronize(s));
            L.launches++;
        }
        L.groups++;
    }
    return DBEEL_OK;
}

// The batches' searches, one level at a time: level j pairs every batch b with its table T_b - 1 - j (newest first).  Per
// level, for all pairs together: one k_gvs_filter; one read-back of the pairs' open-query counts when some pair's fence
// decision needs it; then gvs_level.  Then the entries of hits at fences are read into the heap, k_gvs_hit decodes every
// hit and split_emit writes `out` in query order, as dbeel_get_values does.  Every phase ends in a stream synchronise
// before its pinned buffers are refilled.
// Each pair's decisions are its batch's solo call's: a reader table whose cached fences serve the batch
// (reader_uses_cache) descends them instead of reading its fences; when the depth the batch wants cannot exceed the cached
// one for any number of open queries, the decision is made before the filter and needs no count.
// The caller has checked the arguments, taken the engine and cleared stats and out; results has Σ n_keys rows.
int gvs_walk(dbeel_engine *e, const std::vector<GvsBatch> &bs, dbeel_out *out, dbeel_lookup_result *results) {
    const uint32_t nb = (uint32_t)bs.size();
    uint64_t n_keys = 0;
    std::vector<uint64_t> row0(nb + 1, 0);
    uint32_t levels = 0;
    for (uint32_t b = 0; b < nb; b++) {
        row0[b + 1] = row0[b] + bs[b].n_keys;
        if (bs[b].n_keys) levels = std::max(levels, (uint32_t)bs[b].td.size());
    }
    n_keys = row0[nb];
    if (n_keys == 0) return DBEEL_OK;
    cudaStream_t s = e->stream;
    const uint32_t n = (uint32_t)n_keys;
    const uint64_t budget = e->partition_bytes;
    // the keys of every batch back to back (one batch: as given), and each query's batch
    std::vector<uint8_t> kcat;
    std::vector<uint64_t> ocat;
    std::vector<uint32_t> qb;
    const uint8_t *keys = bs[0].keys;
    const uint64_t *key_off = bs[0].key_off;
    if (nb > 1) {
        ocat.resize(n_keys + 1);
        qb.resize(n_keys);
        for (uint32_t b = 0; b < nb; b++) {
            const GvsBatch &B = bs[b];
            if (!B.n_keys) continue;
            const uint64_t k0 = B.key_off[0], base = kcat.size();
            for (uint64_t i = 0; i < B.n_keys; i++) {
                ocat[row0[b] + i] = base + (B.key_off[i] - k0);
                qb[row0[b] + i] = b;
            }
            kcat.insert(kcat.end(), B.keys + k0, B.keys + B.key_off[B.n_keys]);
        }
        ocat[n_keys] = kcat.size();
        keys = kcat.data();
        key_off = ocat.data();
    }
    const uint64_t key_bytes = key_off[n_keys];
    // the touched flags of a level: at most 2^max(lookup_depth(n_keys), cached depth) per pair
    uint64_t touched_max = 1;
    for (uint32_t j = 0; j < levels; j++) {
        uint64_t t = 0;
        for (const GvsBatch &B : bs) {
            if (!B.n_keys || j >= B.td.size()) continue;
            const uint32_t ti = (uint32_t)B.td.size() - 1 - j;
            const TableDesc &d = B.td[ti];
            uint32_t dmax = lookup_depth(B.n_keys, d.n, d.data_len, 8 + B.max_klen, budget);
            if (B.r) dmax = std::max(dmax, (uint32_t)B.r->tables[ti]->depth);
            t += 1ull << dmax;
        }
        touched_max = std::max(touched_max, t);
    }

    // ---- per-query state and the split's workspace
    uint64_t off = 0;
    const uint64_t o_keys = carve_ws(&off, key_bytes + 16), o_off = carve_ws(&off, 8ull * (n + 1)), o_batch = carve_ws(&off, 4ull * n);
    const uint64_t o_rows = carve_ws(&off, 16ull * n), o_hix = carve_ws(&off, 16ull * n), o_state = carve_ws(&off, sizeof(SearchState) * n);
    const uint64_t o_node = carve_ws(&off, 4ull * n), o_src = carve_ws(&off, 8ull * n), o_hoff = carve_ws(&off, 8ull * n);
    const uint64_t o_touched = carve_ws(&off, touched_max), o_cnt = carve_ws(&off, 8ull * nb), o_need = carve_ws(&off, 8);
    const uint64_t o_cursor = carve_ws(&off, 8), o_pairs = carve_ws(&off, sizeof(GvsPair) * nb);
    const SplitLayout w = carve_split(&off, n, 1);
    int rc = ensure_device(e, &e->ws, &e->ws_cap, off);
    const uint64_t pin_tot = align_up(w.header2_bytes, 64);
    // the pinned block during the levels: touched flags | open counts | the pairs as the filter reads them | as the rest do
    const uint64_t p_cnt = align_up(touched_max, 64), p_fpairs = align_up(p_cnt + 8ull * nb, 64);
    const uint64_t p_pairs = align_up(p_fpairs + sizeof(GvsPair) * nb, 64), p_end = p_pairs + sizeof(GvsPair) * nb;
    if (!rc) rc = ensure_pinned(e, std::max<uint64_t>(pin_tot + 8ull * 4, p_end));
    if (rc) return rc;
    uint8_t *ws = e->ws;
    CU(cudaEventRecord(e->ev[EV_START], s));
    for (uint64_t q = 0; q < n_keys; q++) results[q] = dbeel_lookup_result{-1, 0, 0};
    static_assert(sizeof(dbeel_lookup_result) == 16, "result rows are written as uint4");
    if (key_bytes) CU(cudaMemcpyAsync(ws + o_keys, keys, key_bytes, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ws + o_off, key_off, 8ull * (n + 1), cudaMemcpyHostToDevice, s));
    if (nb > 1) CU(cudaMemcpyAsync(ws + o_batch, qb.data(), 4ull * n, cudaMemcpyHostToDevice, s));
    else CU(cudaMemsetAsync(ws + o_batch, 0, 4ull * n, s));
    CU(cudaMemcpyAsync(ws + o_rows, results, 16ull * n, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(ws + o_src, 0, 8ull * n, s));
    CU(cudaMemsetAsync(ws + o_hoff, 0xFF, 8ull * n, s)); // kGvsNoEntry
    CU(cudaMemsetAsync(ws + o_cursor, 0, 8, s));
    GvsQueries gq{ws + o_keys, reinterpret_cast<const uint64_t *>(ws + o_off), reinterpret_cast<const uint32_t *>(ws + o_batch), n_keys,
                  reinterpret_cast<uint4 *>(ws + o_rows), reinterpret_cast<uint4 *>(ws + o_hix), reinterpret_cast<SearchState *>(ws + o_state),
                  reinterpret_cast<uint32_t *>(ws + o_node), reinterpret_cast<unsigned long long *>(ws + o_src),
                  reinterpret_cast<unsigned long long *>(ws + o_hoff)};
    GvsLevel L{gq, (n + 255) / 256, reinterpret_cast<GvsPair *>(ws + o_pairs), ws + o_touched, p_pairs,
               reinterpret_cast<unsigned long long *>(ws + o_need), reinterpret_cast<unsigned long long *>(ws + o_cursor)};
    unsigned long long *d_cnt = reinterpret_cast<unsigned long long *>(ws + o_cnt);

    std::vector<GvsPair> pairs(nb);
    std::vector<LeafSrc> src(nb);
    std::vector<uint64_t> count(nb);
    for (uint32_t j = 0; j < levels; j++) {
        // ---- the filter, with the decisions that need no count of open queries: the depth the batch wants grows with
        // that count, which is at most its n_keys
        std::vector<const ProbeTree *> pts(nb, nullptr);
        bool need_count = false;
        for (uint32_t b = 0; b < nb; b++) {
            const GvsBatch &B = bs[b];
            GvsPair &P = pairs[b];
            P = GvsPair{};
            P.mode = B.mode;
            src[b] = LeafSrc{B.r, B.io, 0, 0, B.max_klen};
            if (!B.n_keys || j >= B.td.size()) continue;
            const uint32_t ti = (uint32_t)B.td.size() - 1 - j;
            P.t = B.td[ti];
            P.table = ti;
            P.live = 1;
            src[b].table = ti;
            src[b].data_len = P.t.data_len;
            dbeel_reader_table *rt = B.r ? B.r->tables[ti].get() : nullptr;
            dbeel_reader_table::Fences *cache = rt ? &rt->fences[B.mode] : nullptr;
            const uint32_t cd = rt ? (uint32_t)rt->depth : 0;
            if (cache && cache->loaded && cd > 0 &&
                reader_uses_cache(B.max_klen, lookup_depth(B.n_keys, P.t.n, P.t.data_len, 8 + B.max_klen, budget), cd)) {
                P.depth = cd;
                pts[b] = &cache->pt;
                P.fix = reinterpret_cast<const uint4 *>(cache->dev);
                P.ffr = reinterpret_cast<const unsigned long long *>(cache->dev + (16ull << cd));
            } else {
                need_count = true;
            }
        }
        memcpy(e->pin + p_fpairs, pairs.data(), sizeof(GvsPair) * nb);
        CU(cudaMemcpyAsync(L.d_pairs, e->pin + p_fpairs, sizeof(GvsPair) * nb, cudaMemcpyHostToDevice, s));
        CU(cudaMemsetAsync(d_cnt, 0, 8ull * nb, s));
        launch_k(e, k_gvs_filter, L.grid, 256, 0, s, gq, static_cast<const GvsPair *>(L.d_pairs), d_cnt);
        L.launches++;
        if (need_count) {
            CU(cudaMemcpyAsync(e->pin + p_cnt, d_cnt, 8ull * nb, cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
            memcpy(count.data(), e->pin + p_cnt, 8ull * nb);
        }
        if ((rc = gvs_level<false>(e, L, pairs, src, count, pts))) return rc;
    }

    // ---- hits at fences: their entries, one record each (runs that touch as one read), per pair into the heap behind
    // the copies
    std::vector<uint4> hix(n);
    std::vector<unsigned long long> hoff(n);
    CU(cudaMemcpyAsync(results, ws + o_rows, 16ull * n, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(hix.data(), ws + o_hix, 16ull * n, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(hoff.data(), ws + o_hoff, 8ull * n, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    std::vector<uint32_t> pair0(nb + 1, 0); // batch b's tables are pairs [pair0[b], pair0[b + 1]) of the entry reads
    for (uint32_t b = 0; b < nb; b++) pair0[b + 1] = pair0[b] + (uint32_t)bs[b].td.size();
    std::vector<std::vector<ByteRange>> er(pair0[nb]);
    auto fence_entry = [&](uint32_t b, uint64_t q, ByteRange *r) { // a fence hit whose entry k_gvs_hit can decode
        if (hoff[q] != kGvsFenceHit) return false;
        const uint4 ix = hix[q];
        const uint64_t o = (uint64_t)ix.x | ((uint64_t)ix.y << 32), dl = bs[b].td[results[q].table].data_len;
        if (!gvs_entry_fits(o, ix.z, ix.w, key_off[q + 1] - key_off[q], dl)) return false;
        *r = ByteRange{o, o + ix.w};
        return true;
    };
    bool any_fence_hit = false;
    for (uint32_t b = 0; b < nb; b++)
        for (uint64_t q = row0[b]; q < row0[b + 1]; q++) {
            ByteRange r;
            if (fence_entry(b, q, &r)) er[pair0[b] + results[q].table].push_back(r);
            any_fence_hit = any_fence_hit || hoff[q] == kGvsFenceHit;
        }
    if (any_fence_hit) {
        const uint64_t base = align_up(L.heap_bound, kAlign);
        std::vector<GvsStaged> sh(pair0[nb]);
        std::vector<GvsPart> parts;
        uint64_t staged = 0;
        for (uint32_t b = 0; b < nb; b++)
            for (uint32_t i = 0; i < bs[b].td.size(); i++) {
                GvsStaged &x = sh[pair0[b] + i];
                x = gvs_stage(std::move(er[pair0[b] + i]), 0, staged);
                staged = x.end;
                if (!x.runs.empty()) parts.push_back(GvsPart{i, &x, bs[b].r, bs[b].io});
            }
        if ((rc = ensure_host(e, &e->ring_in, &e->ring_in_cap, std::max<uint64_t>(staged, 256)))) return rc;
        if ((rc = gvs_heap_reserve(e, base + staged + 256, L.heap_bound))) return rc;
        if ((rc = gvs_load(e, DBEEL_STREAM_DATA, parts, e->ring_in, e->stage_out2 + base, 0, staged, false, "stream read callback failed (.data, entries)")))
            return rc;
        for (uint32_t b = 0; b < nb; b++)
            for (uint64_t q = row0[b]; q < row0[b + 1]; q++) {
                ByteRange r;
                if (hoff[q] != kGvsFenceHit) continue;
                hoff[q] = fence_entry(b, q, &r) ? base + sh[pair0[b] + results[q].table].at(r.lo) : kGvsNoEntry;
            }
        CU(cudaMemcpyAsync(ws + o_hoff, hoff.data(), 8ull * n, cudaMemcpyHostToDevice, s));
        CU(cudaStreamSynchronize(s));
    }
    ScanParams sp = {};
    RouteParams rp;
    Params p;
    split_bind(w, ws, &sp, &rp, &p);
    CU(cudaMemsetAsync(ws + w.o_tot, 0, 8ull * 3, s));
    CU(cudaMemsetAsync(sp.stop, 0xFF, 8, s));
    launch_k(e, k_gvs_hit, L.grid, 256, 0, s, gq, static_cast<const uint8_t *>(e->stage_out2), LookupEmit{sp.dest, sp.flat});
    L.launches++;
    CU(cudaMemcpyAsync(results, ws + o_rows, 16ull * n, cudaMemcpyDeviceToHost, s)); // back with the sizes: filled on ERR_CAPACITY too
    e->stats.entries_in = n_keys;
    e->stats.partitions = L.groups;
    uint64_t items = 0, bytes = 0;
    rc = split_emit(e, w, sp, rp, p, pin_tot, false, out, &L.launches, &items, &bytes, [](const unsigned long long *) {});
    if (rc == DBEEL_ERR_CAPACITY) {
        out->data_len = bytes;
        out->index_len = 16 * items;
        return fail(e, DBEEL_ERR_CAPACITY, "the entries found are larger than the output buffers (data_len / index_len: the sizes needed)");
    }
    return rc;
}

// dbeel_get_values_stream and dbeel_reader_get_values: one batch.
int get_values_stream_entry(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys, const uint64_t *key_off,
                            uint64_t n_keys, uint32_t mode, const dbeel_scan_io *io, dbeel_out *out, dbeel_lookup_result *results,
                            dbeel_reader *reader = nullptr) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || !io || !io->read) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (const int arc = lookup_args(e, tables, n_tables, key_off, n_keys, mode, results)) return arc;
    if (n_keys >= 0xFFFFFFF0ull) return fail(e, DBEEL_ERR_INVALID_ARG, "2^32 - 16 keys or more");
    const Claim c(e);
    if (c.rc) return c.rc;
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    if (n_keys == 0) return DBEEL_OK;
    for (uint32_t i = 0; i < n_tables; i++) { // as stage_lookup; .data and .index come through the callback
        const dbeel_table &t = tables[i];
        if (t.index_len % DBEEL_INDEX_ENTRY_SIZE) return fail(e, DBEEL_ERR_INVALID_ARG, "index length is not a multiple of 16");
        if (t.bloom_len && !t.bloom) return fail(e, DBEEL_ERR_INVALID_ARG, "null table buffer");
        if (t.bloom_len && (t.bloom_len < 8 + kBloomTrailer || (t.bloom_len - 8 - kBloomTrailer) % 4))
            return fail(e, DBEEL_ERR_BAD_BLOOM, "bloom file length is not 8 + 4 * words + 164");
    }
    const uint64_t key_bytes = key_off[n_keys];
    if (!keys && key_bytes) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    int rc;
    uint64_t bloom_bytes = 0;
    for (uint32_t i = 0; i < n_tables; i++) bloom_bytes += align_up(tables[i].bloom_len + 16, kAlign);
    if ((rc = ensure_device(e, &e->bloom_dev, &e->bloom_dev_cap, std::max<uint64_t>(bloom_bytes, 256)))) return rc;
    std::vector<GvsBatch> bs(1);
    GvsBatch &B = bs[0];
    B.r = reader;
    B.io = io;
    B.keys = static_cast<const uint8_t *>(keys);
    B.key_off = key_off;
    B.n_keys = n_keys;
    B.mode = mode;
    for (uint64_t q = 0; q < n_keys; q++) B.max_klen = std::max(B.max_klen, key_off[q + 1] - key_off[q]);
    B.td.resize(n_tables);
    uint64_t bpos = 0;
    for (uint32_t i = 0; i < n_tables; i++) {
        const dbeel_table &t = tables[i];
        B.td[i] = TableDesc{nullptr, t.data_len, nullptr, t.index_len / DBEEL_INDEX_ENTRY_SIZE, nullptr, 0, 0, 0, 0, {0, 0, 0, 0}};
        if (reader) B.td[i] = reader->tables[i]->desc; // tables[] carries no filter: it is resident
        if (!t.bloom_len) continue;
        const uint8_t *b = static_cast<const uint8_t *>(t.bloom);
        if ((rc = parse_bloom(e, b, b + t.bloom_len - kBloomTrailer, t.bloom_len, &B.td[i]))) return rc;
        CU(cudaMemcpyAsync(e->bloom_dev + bpos, b, t.bloom_len, cudaMemcpyHostToDevice, e->stream));
        B.td[i].words = reinterpret_cast<const uint32_t *>(e->bloom_dev + bpos + 8);
        bpos += align_up(t.bloom_len + 16, kAlign);
    }
    return gvs_walk(e, bs, out, results);
}


// ------------------------------------------------------------------------------------ N5 streamed: dbeel_scan_stream
// The plan (host/scan_plan.h) cuts the record sequence into partitions; each goes file -> pinned ring slot -> device slot
// c & 1 in ONE H2D copy of its slot image (table headers | per slice: index slice, .data window), runs k_scan_classify,
// launch_split, k_scan_stream_carry and launch_phase2 with phase 2 sized from the plan's bound (the split's workspace from
// split_bind, as split_emit's), and comes back with an exact D2H of what it selected.  H2D of c + 1, the kernels of c
// and the D2H of c - 1 overlap; the engine thread enqueues partition c + 1's kernels before it waits for c's published sizes.
// run_scan_plan runs a plan (steps 2 to the end) for dbeel_scan_stream (whole tables) and dbeel_reader_scan (spans): the
// caller has checked the arguments, taken the engine, cleared results / stop / stats and set stats.entries_in.
// dbeel_reader_get_range passes `merge` (a key-aligned plan, plan_merge): every partition runs the merge stage of
// merge_range.cuh between the split and phase 2, and merge->unsorted reports a table whose span records do not ascend.
struct RangeMerge {
    const std::vector<std::vector<uint8_t>> *cuts; // plan.parts.size() - 1 ascending splitters (MergePlan::cuts)
    bool keep_tombstones;
    bool unsorted; // out
};

int run_scan_plan(dbeel_engine *e, const dbeel_table *tables, const ScanPlan &plan, uint32_t kind, const void *ranges,
                  uint32_t n_ranges, uint64_t key_bytes, const dbeel_scan_io *io, dbeel_job_result *results, dbeel_scan_stop *stop,
                  RangeMerge *merge = nullptr) {
    int rc = DBEEL_OK;
    const uint32_t np = (uint32_t)plan.parts.size();
    e->stats.partitions = np;
    auto host_stop = [&]() {
        if (plan.panic_table >= 0) *stop = dbeel_scan_stop{plan.panic_table, DBEEL_SCAN_STOP_PANIC, plan.panic_record};
    };
    if (np == 0) { host_stop(); return DBEEL_OK; }
    cudaStream_t s = e->stream;

    // ---- 2. slot layouts: [ScanTable per slice | per slice: index slice (+16), .data window (+32)], 256-byte aligned pieces
    auto slot_layout = [&](uint32_t c, auto &&fn) { // fn(slice, index position, window position); returns the slot's bytes
        const ScanPart &pt = plan.parts[c];
        uint64_t pos = align_up(sizeof(ScanTable) * pt.n_slices, kAlign);
        for (uint32_t k = 0; k < pt.n_slices; k++) {
            const ScanSlice &sl = plan.slices[pt.first_slice + k];
            const uint64_t ip = pos;
            pos += align_up(16 * (sl.rec_hi - sl.rec_lo) + 16, kAlign);
            fn(k, sl, ip, pos);
            pos += align_up(sl.win_hi - sl.win_lo + 32, kAlign);
        }
        return pos;
    };
    const uint32_t nd = n_ranges;
    uint64_t max_in = 0, max_rec = 0, max_bound = 0, h2d_bytes = 0;
    for (uint32_t c = 0; c < np; c++) {
        const uint64_t in = slot_layout(c, [](uint32_t, const ScanSlice &, uint64_t, uint64_t) {});
        max_in = std::max(max_in, in);
        max_rec = std::max(max_rec, plan.parts[c].n_rec);
        max_bound = std::max(max_bound, plan.parts[c].data_bound);
        h2d_bytes += in;
    }
    const uint64_t out_index_at = align_up(max_bound + 16, kAlign), max_out = out_index_at + align_up(16 * max_rec + 16, kAlign);
    const uint64_t gather_tiles_max = (max_bound + kGatherTileBytes - 1) / kGatherTileBytes;
    uint64_t off = 0;
    const RangeHeader rh = carve_ranges(&off, kind, nd, key_bytes);
    const SplitLayout w = carve_split(&off, (uint32_t)max_rec, nd);
    const uint64_t o_carry = carve_ws(&off, 8ull * (2 * nd + 1)), o_tf = carve_ws(&off, 4ull * (gather_tiles_max + 2));
    const uint64_t pub_words = 5ull * nd + 2, pub_stride = align_up(8 * pub_words, 64), pin_pub = align_up(rh.bytes, 64);
    // the merge stage: per split record its table, key prefix and keep flag / prefix sum; per destination its surviving
    // bytes; the error word; every slice's table and every splitter, uploaded once
    std::vector<uint32_t> m_slt;
    std::vector<uint64_t> m_koff(1, 0);
    std::vector<uint8_t> m_keys;
    uint64_t o_mtab = 0, o_mpfx = 0, o_mpre = 0, o_mtile = 0, o_mbytes = 0, o_merr = 0, o_mslt = 0, o_mkeys = 0;
    if (merge) {
        for (const ScanSlice &sl : plan.slices) m_slt.push_back(sl.table);
        for (const std::vector<uint8_t> &k : *merge->cuts) {
            m_keys.insert(m_keys.end(), k.begin(), k.end());
            m_koff.push_back(m_keys.size());
        }
        o_mtab = carve_ws(&off, 4ull * w.n);
        o_mpfx = carve_ws(&off, 8ull * w.n);
        o_mpre = carve_ws(&off, 4ull * w.n + 4);
        o_mtile = carve_ws(&off, 4ull * ((w.n + kRangeTile - 1) / kRangeTile + 1));
        o_mbytes = carve_ws(&off, 8ull * nd);
        o_merr = carve_ws(&off, 8);
        o_mslt = carve_ws(&off, 4ull * m_slt.size());
        o_mkeys = carve_ws(&off, m_keys.size() + 16);
    }
    const uint32_t R = (uint32_t)std::max(2, e->stream_ring);
    rc = ensure_device(e, &e->ws, &e->ws_cap, off);
    if (!rc) rc = ensure_device(e, &e->stage_in, &e->stage_in_cap, max_in);
    if (!rc) rc = ensure_device(e, &e->stage_in2, &e->stage_in2_cap, max_in);
    if (!rc) rc = ensure_device(e, &e->stage_out, &e->stage_out_cap, max_out);
    if (!rc) rc = ensure_device(e, &e->stage_out2, &e->stage_out2_cap, max_out);
    if (!rc) rc = ensure_pinned(e, pin_pub + 2 * pub_stride);
    if (!rc) rc = ensure_host(e, &e->ring_in, &e->ring_in_cap, (uint64_t)R * max_in);
    if (!rc) rc = ensure_host(e, &e->ring_out, &e->ring_out_cap, (uint64_t)R * max_out);
    if (!rc) rc = ensure_copy_streams(e);
    if (rc) return rc;
    uint8_t *ws = e->ws;
    uint8_t *sin[2] = {e->stage_in, e->stage_in2}, *sout[2] = {e->stage_out, e->stage_out2};

    // ---- 3. the pump: every partition's index slices and windows into its ring slot, the outputs to the write callback
    struct EventList {
        std::vector<cudaEvent_t> ev;
        ~EventList() { for (auto &x : ev) if (x) cudaEventDestroy(x); }
    } ev_out;
    ev_out.ev.assign(np, nullptr);
    for (uint32_t c = 0; c < np; c++) CU(cudaEventCreateWithFlags(&ev_out.ev[c], cudaEventDisableTiming | cudaEventBlockingSync));
    const int dev = e->device;
    EventList *evl = &ev_out;
    StreamPump pump(io, np, R, stream_threads(), [evl](uint32_t c) { cudaEventSynchronize(evl->ev[c]); }, [dev]() { cudaSetDevice(dev); });
    for (uint32_t c = 0; c < np; c++) {
        uint8_t *slot = e->ring_in + (uint64_t)(c % R) * max_in;
        slot_layout(c, [&](uint32_t, const ScanSlice &sl, uint64_t ip, uint64_t wp) {
            pump.add_read(c, sl.table, DBEEL_STREAM_INDEX, 16 * sl.rec_lo, 16 * (sl.rec_hi - sl.rec_lo), slot + ip);
            pump.add_read(c, sl.table, DBEEL_STREAM_DATA, sl.win_lo, sl.win_hi - sl.win_lo, slot + wp);
        });
    }
    pump.start();

    // ---- 4. per-scan state on the device: ranges (once), carry, stop word.  stop0 stays none: the plan ends before every
    // stop the index shows (empty tables included).
    ScanParams sp = {};
    RouteParams rp;
    Params p;
    split_bind(w, ws, &sp, &rp, &p);
    p.tile_first = reinterpret_cast<uint32_t *>(ws + o_tf);
    unsigned long long *carry = reinterpret_cast<unsigned long long *>(ws + o_carry);
    CU(cudaEventRecord(e->ev[EV_START], s));
    land_ranges(e, rh, kind, ranges, nd, key_bytes, &sp);
    CU(cudaMemsetAsync(carry, 0, 8ull * (2 * nd + 1), s));
    CU(cudaMemsetAsync(sp.stop, 0xFF, 8, s));
    RangeMergeParams mp = {};
    if (merge) {
        CU(cudaMemsetAsync(ws + o_mbytes, 0, 8ull * nd, s));
        CU(cudaMemsetAsync(ws + o_merr, 0, 8, s));
        CU(cudaMemcpyAsync(ws + o_mslt, m_slt.data(), 4ull * m_slt.size(), cudaMemcpyHostToDevice, s));
        if (!m_keys.empty()) CU(cudaMemcpyAsync(ws + o_mkeys, m_keys.data(), m_keys.size(), cudaMemcpyHostToDevice, s));
        mp.n_ranges = nd;
        mp.keep_tombstones = merge->keep_tombstones ? 1u : 0u;
        mp.flat = sp.flat;
        mp.split = rp.out_index;
        mp.out = sp.flat;
        mp.totals = rp.totals;
        mp.tab = reinterpret_cast<uint32_t *>(ws + o_mtab);
        mp.pfx = reinterpret_cast<unsigned long long *>(ws + o_mpfx);
        mp.pre = reinterpret_cast<uint32_t *>(ws + o_mpre);
        mp.tile = reinterpret_cast<uint32_t *>(ws + o_mtile);
        mp.dbytes = reinterpret_cast<unsigned long long *>(ws + o_mbytes);
        mp.err = reinterpret_cast<uint32_t *>(ws + o_merr);
    }

    // ---- 5. the pipeline
    auto enqueue_h2d = [&](uint32_t c) -> int {
        const int prc = pump.wait_reads(c);
        if (prc) return fail(e, prc, "stream read callback failed");
        uint8_t *slot = e->ring_in + (uint64_t)(c % R) * max_in, *base = sin[c & 1];
        ScanTable *td = reinterpret_cast<ScanTable *>(slot);
        uint32_t local = 0;
        const uint64_t bytes = slot_layout(c, [&](uint32_t k, const ScanSlice &sl, uint64_t ip, uint64_t wp) {
            const uint32_t nr = (uint32_t)(sl.rec_hi - sl.rec_lo);
            // biased: .data offset `off` of the table lives at data + off, inside the window
            td[k] = ScanTable{reinterpret_cast<const uint8_t *>(reinterpret_cast<uintptr_t>(base + wp) - sl.win_lo), tables[sl.table].data_len,
                              reinterpret_cast<const uint4 *>(base + ip), nr, local};
            local += nr;
        });
        CU(cudaMemcpyAsync(base, slot, bytes, cudaMemcpyHostToDevice, e->s_h2d));
        CU(cudaEventRecord(e->ev_h2d[c & 1], e->s_h2d));
        return DBEEL_OK;
    };
    uint32_t launches = 0;
    auto enqueue_kernels = [&](uint32_t c) -> int {
        const ScanPart &pt = plan.parts[c];
        const uint32_t n = (uint32_t)pt.n_rec, nb = (n + kRouteThreads - 1) / kRouteThreads;
        const uint64_t gtiles = (pt.data_bound + kGatherTileBytes - 1) / kGatherTileBytes;
        CU(cudaStreamWaitEvent(s, e->ev_h2d[c & 1], 0));
        if (c >= 2) CU(cudaStreamWaitEvent(s, e->ev_d2h[c & 1], 0)); // output slot c & 1 has gone back to the host
        ScanParams spc = sp;
        spc.tables = reinterpret_cast<const ScanTable *>(sin[c & 1]);
        spc.n_tables = pt.n_slices;
        spc.n = n;
        RouteParams rpc = rp;
        rpc.n = n;
        rpc.n_blocks = nb;
        Params pc = p;
        pc.tile_first_n = (uint32_t)(gtiles + 2);
        pc.data_bound = pt.data_bound;
        pc.out_data = sout[c & 1];
        pc.out_index = reinterpret_cast<uint4 *>(sout[c & 1] + out_index_at);
        unsigned long long *pub = reinterpret_cast<unsigned long long *>(e->pin_dev + pin_pub + (c & 1) * pub_stride);
        CU(cudaMemsetAsync(rp.totals, 0, 8ull * 3 * nd, s));
        launch_k(e, k_scan_classify, (n + 255) / 256, 256, 0, s, spc);
        launch_split(e, spc, rpc, pub);
        const uint4 *split = rpc.out_index;
        if (merge) { // the merged split replaces the split, in flat
            RangeMergeParams mpc = mp;
            mpc.tables = spc.tables;
            mpc.slice_table = reinterpret_cast<const uint32_t *>(ws + o_mslt) + pt.first_slice;
            mpc.n_slices = pt.n_slices;
            mpc.n = n;
            mpc.pub = pub;
            if (c > 0) {
                mpc.lo = ws + o_mkeys + m_koff[c - 1];
                mpc.lo_len = (uint32_t)(m_koff[c] - m_koff[c - 1]);
            }
            if (c + 1 < np) {
                mpc.hi = ws + o_mkeys + m_koff[c];
                mpc.hi_len = (uint32_t)(m_koff[c + 1] - m_koff[c]);
            }
            const uint32_t g = (n + 255) / 256, gt = (n + kRangeTile - 1) / kRangeTile;
            launch_k(e, k_range_keys, g, 256, 0, s, mpc);
            launch_k(e, k_range_check, g, 256, 0, s, mpc);
            launch_k(e, k_range_flag, g, 256, 0, s, mpc);
            launch_k(e, k_range_tile_sums, gt, kRangeTile, 0, s, mpc);
            launch_k(e, k_range_tile_scan, 1, kRangeTile, 0, s, mpc);
            launch_k(e, k_range_prefix, gt, kRangeTile, 0, s, mpc);
            launch_k(e, k_range_rank, g, 256, 0, s, mpc);
            launch_k(e, k_range_totals, 1, 256, 0, s, mpc);
            launches += 8;
            split = sp.flat;
        }
        launch_k(e, k_scan_stream_carry, 1, 32, 0, s, rpc, pc, carry, pub);
        launch_phase2(e, pc, split, n, gtiles);
        launches += 12;
        CU(cudaGetLastError());
        CU(cudaEventRecord(e->ev_comp[c & 1], s));
        return DBEEL_OK;
    };
    uint64_t out_bytes = 0;
    std::vector<unsigned long long> hdr(pub_words);
    bool stopped = false;
    rc = enqueue_h2d(0);
    if (!rc && np > 1) rc = enqueue_h2d(1);
    if (!rc) rc = enqueue_kernels(0);
    for (uint32_t c = 0; c < np && !rc; c++) {
        if (c + 1 < np) {
            rc = enqueue_kernels(c + 1);
            if (rc) break;
        }
        const cudaError_t ce = cudaEventSynchronize(e->ev_comp[c & 1]);
        if (ce != cudaSuccess) { rc = fail(e, DBEEL_ERR_CUDA, "scan kernels", ce); break; }
        pump.release_input(c); // H2D c (out of ring slot c mod R) has completed
        memcpy(hdr.data(), e->pin + pin_pub + (c & 1) * pub_stride, 8 * pub_words);
        // counts | bytes | starts | stop | carry bytes | carry entries | halted before this partition
        const ScanPart &pt = plan.parts[c];
        if (!hdr[5 * nd + 1] && hdr[3 * nd] != ~0ull && !stopped) {
            const unsigned long long key = hdr[3 * nd];
            const uint32_t lt = (uint32_t)((key >> 2) & 1023);
            uint64_t local = 0;
            for (uint32_t k = 0; k < lt; k++) local += plan.slices[pt.first_slice + k].rec_hi - plan.slices[pt.first_slice + k].rec_lo;
            const ScanSlice &sl = plan.slices[pt.first_slice + lt];
            *stop = dbeel_scan_stop{(int32_t)sl.table, (uint32_t)(key & 3), sl.rec_lo + ((key >> 12) - local)};
            stopped = true;
        }
        uint64_t bytes = 0, items = 0;
        for (uint32_t d = 0; d < nd; d++) { bytes += hdr[nd + d]; items += hdr[d]; }
        rc = pump.wait_out_slot(c);
        if (rc) { fail(e, rc, "stream write callback failed"); break; }
        uint8_t *oslot = e->ring_out + (uint64_t)(c % R) * max_out;
        CU(cudaStreamWaitEvent(e->s_d2h, e->ev_comp[c & 1], 0));
        if (bytes) CU(cudaMemcpyAsync(oslot, sout[c & 1], bytes, cudaMemcpyDeviceToHost, e->s_d2h));
        if (items) CU(cudaMemcpyAsync(oslot + out_index_at, sout[c & 1] + out_index_at, 16 * items, cudaMemcpyDeviceToHost, e->s_d2h));
        CU(cudaEventRecord(ev_out.ev[c], e->s_d2h));
        CU(cudaEventRecord(e->ev_d2h[c & 1], e->s_d2h));
        std::vector<StreamPump::OutPiece> pieces;
        uint64_t before = 0; // destination d's bytes start here in the partition's output (its entries at starts[d])
        for (uint32_t d = 0; d < nd; d++) {
            const uint64_t db = hdr[nd + d], di = hdr[d];
            if (di) {
                pieces.push_back({d, DBEEL_STREAM_DATA, hdr[3 * nd + 1 + d], oslot + before, db});
                pieces.push_back({d, DBEEL_STREAM_INDEX, 16 * hdr[4 * nd + 1 + d], oslot + out_index_at + 16 * hdr[2 * nd + d], 16 * di});
            }
            before += db;
            results[d].data_len += db;
            results[d].items_written += di;
        }
        out_bytes += bytes + 16 * items;
        pump.publish_pieces(c, std::move(pieces));
        if (c + 2 < np) rc = enqueue_h2d(c + 2);
    }
    if (rc) { // drain: nothing of this scan may touch the engine's buffers after it returns
        cudaStreamSynchronize(e->s_h2d);
        cudaStreamSynchronize(s);
        cudaStreamSynchronize(e->s_d2h);
        pump.abort(rc);
        clear_scan(results, nd, stop);
        return rc;
    }
    CU(cudaEventRecord(e->ev[EV_GATHER], s));
    CU(cudaStreamSynchronize(s));
    CU(cudaStreamSynchronize(e->s_d2h));
    const int frc = pump.finish(); // every destination's bytes have gone through the write callback
    if (frc) {
        clear_scan(results, nd, stop);
        return fail(e, frc, "stream write callback failed");
    }
    if (!stopped) host_stop();
    if (merge) {
        uint32_t err = 0;
        CU(cudaMemcpy(&err, ws + o_merr, 4, cudaMemcpyDeviceToHost));
        merge->unsorted = err != 0;
    }
    uint64_t items = 0;
    for (uint32_t d = 0; d < nd; d++) {
        results[d].index_len = 16 * results[d].items_written;
        items += results[d].items_written;
    }
    cudaEventElapsedTime(&e->stats.ms_total, e->ev[EV_START], e->ev[EV_GATHER]);
    e->stats.kernel_launches = launches + 1;
    e->stats.input_bytes = h2d_bytes;
    e->stats.output_bytes = out_bytes;
    e->stats.entries_out = items;
    return DBEEL_OK;
}

// The tables as plan_scan / plan_merge take them: their lengths, and their .index files read through io->read.
struct PlanTables {
    std::vector<uint64_t> dlen, ilen;
    ScanIndexRead read_index;
};

PlanTables plan_tables(const dbeel_table *tables, uint32_t n_tables, const dbeel_scan_io *io) {
    PlanTables pt{std::vector<uint64_t>(n_tables), std::vector<uint64_t>(n_tables),
                  [io](uint32_t t, uint64_t off, uint64_t len, void *dst) { return io->read(io->ctx, t, DBEEL_STREAM_INDEX, off, len, dst); }};
    for (uint32_t t = 0; t < n_tables; t++) {
        pt.dlen[t] = tables[t].data_len;
        pt.ilen[t] = tables[t].index_len;
    }
    return pt;
}

// 1. plan_scan over tables[0 .. n_tables) through io->read, from the .index files read in pieces; then run_scan_plan.
// spans: null = whole tables, whose index records all count in stats.entries_in (reader_spans counts the spans').
int plan_and_run_scan(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges,
                      uint32_t n_ranges, uint64_t key_bytes, const dbeel_scan_io *io, dbeel_job_result *results,
                      dbeel_scan_stop *stop, const std::vector<std::vector<ScanSpan>> *spans) {
    if (!spans)
        for (uint32_t t = 0; t < n_tables; t++) e->stats.entries_in += tables[t].index_len / DBEEL_INDEX_ENTRY_SIZE;
    const PlanTables pt = plan_tables(tables, n_tables, io);
    ScanPlan plan;
    const int rc = plan_scan(pt.dlen.data(), pt.ilen.data(), n_tables, e->partition_bytes, pt.read_index, &plan, spans);
    if (rc) return fail(e, rc, "stream read callback failed (.index, planning)");
    return run_scan_plan(e, tables, plan, kind, ranges, n_ranges, key_bytes, io, results, stop);
}

int scan_stream_entry(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges,
                      uint32_t n_ranges, const dbeel_scan_io *io, dbeel_job_result *results, dbeel_scan_stop *stop) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!io || !io->read || !io->write) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    uint64_t key_bytes = 0;
    if (const int arc = scan_args(e, tables, n_tables, kind, ranges, n_ranges, results, stop, &key_bytes)) return arc;
    const Claim c(e);
    if (c.rc) return c.rc;
    clear_scan(results, n_ranges, stop);
    return plan_and_run_scan(e, tables, n_tables, kind, ranges, n_ranges, key_bytes, io, results, stop, nullptr);
}

// ---- dbeel_reader_scan
// The reader's read callback, counted (input_bytes), and the caller's write callback, behind one ctx.
struct ReaderScanIo {
    const dbeel_scan_io *rio;
    int (*write)(void *, uint32_t, uint32_t, uint64_t, const void *, uint64_t);
    void *wctx;
    std::atomic<uint64_t> bytes{0};
};

int reader_scan_read(void *ctx, uint32_t t, uint32_t kind, uint64_t off, uint64_t len, void *dst) {
    ReaderScanIo *x = static_cast<ReaderScanIo *>(ctx);
    x->bytes += len;
    return x->rio->read(x->rio->ctx, t, kind, off, len, dst);
}

int reader_scan_write(void *ctx, uint32_t d, uint32_t kind, uint64_t off, const void *src, uint64_t len) {
    ReaderScanIo *x = static_cast<ReaderScanIo *>(ctx);
    return x->write(x->wctx, d, kind, off, src, len);
}

// The reader's tables as the entry points take them: lengths only, their bytes come through the reader's callback.
std::vector<dbeel_table> reader_tables(const dbeel_reader *r) {
    std::vector<dbeel_table> tables(r->tables.size());
    for (size_t i = 0; i < tables.size(); i++) {
        const TableDesc &d = r->tables[i]->desc;
        tables[i] = dbeel_table{nullptr, d.data_len, nullptr, d.n * DBEEL_INDEX_ENTRY_SIZE, nullptr, 0};
    }
    return tables;
}

// Vec<u8>::cmp(a, b) < 0
inline bool key_less(const uint8_t *a, uint64_t al, const uint8_t *b, uint64_t bl) {
    const int c = std::min(al, bl) ? memcmp(a, b, std::min(al, bl)) : 0;
    return c < 0 || (c == 0 && al < bl);
}

// One reader's part of a seek: seek_t(bound) of dbeel_reader_scan (dbeel_compact.h) for every table t < nseek of r and every
// bound b of kb[boff[b] .. + blen[b]), through io; res / bad / bix[t * nb + b] = the search's result (~0: it failed), its
// corrupt probe (~0: none) and that probe's index record.
struct SeekPart {
    dbeel_reader *r;
    const dbeel_scan_io *io;
    uint32_t nseek;
    const uint8_t *kb;
    std::vector<uint64_t> boff, blen;
    uint64_t depth_queries; // the open queries every pair counts, which size its fences (lookup_depth)
    std::vector<unsigned long long> res, bad;
    std::vector<uint4> bix;
};

// The parts' bound searches as one level of gvs_level<true>: part i's table t is a pair, reader table t in
// DBEEL_LOOKUP_EXACT (its exact-mode fence cache) with no filter, with the part's depth_queries and longest bound, so that
// the depth and cache decisions are each part's own; query t * nb + b of a part searches its pair t.
int reader_seek(dbeel_engine *e, std::vector<SeekPart> &sp) {
    uint64_t Q = 0;
    uint32_t np = 0;
    for (const SeekPart &x : sp) {
        Q += x.boff.size() * x.nseek;
        np += x.nseek;
    }
    if (!Q) return DBEEL_OK;
    cudaStream_t s = e->stream;
    const uint64_t budget = e->partition_bytes;
    // the bounds once per table, so that query q's key is keys[ko[q] .. ko[q + 1])
    std::vector<uint8_t> keys;
    std::vector<uint64_t> ko(Q + 1), count;
    std::vector<uint32_t> qt(Q);
    std::vector<GvsPair> pairs;
    std::vector<LeafSrc> src;
    uint64_t touched_max = 0; // at most 2^max(lookup_depth, cached depth) per pair
    for (uint64_t i = 0, q = 0; i < sp.size(); i++) {
        const SeekPart &x = sp[i];
        const uint64_t nb = x.boff.size();
        uint64_t max_klen = 0;
        for (uint64_t b = 0; b < nb; b++) max_klen = std::max(max_klen, x.blen[b]);
        for (uint32_t t = 0; t < x.nseek; t++) {
            for (uint64_t b = 0; b < nb; b++, q++) {
                ko[q] = keys.size();
                qt[q] = (uint32_t)pairs.size();
                keys.insert(keys.end(), x.kb + x.boff[b], x.kb + x.boff[b] + x.blen[b]);
            }
            const TableDesc &d = x.r->tables[t]->desc;
            pairs.push_back(GvsPair{d, nullptr, nullptr, nullptr, 0, t, DBEEL_LOOKUP_EXACT, 1});
            pairs.back().t.words = nullptr;
            src.push_back(LeafSrc{x.r, x.io, t, d.data_len, max_klen});
            count.push_back(x.depth_queries);
            touched_max += 1ull << std::max(lookup_depth(x.depth_queries, d.n, d.data_len, 8 + max_klen, budget), (uint32_t)x.r->tables[t]->depth);
        }
    }
    ko[Q] = keys.size();

    // ---- per-query state; the pinned block: touched flags | the pairs as the filter reads them | as the rest do
    uint64_t off = 0;
    const uint64_t o_keys = carve_ws(&off, keys.size() + 16), o_off = carve_ws(&off, 8 * (Q + 1)), o_batch = carve_ws(&off, 4 * Q);
    const uint64_t o_rows = carve_ws(&off, 16 * Q), o_hix = carve_ws(&off, 16 * Q), o_state = carve_ws(&off, sizeof(SearchState) * Q);
    const uint64_t o_node = carve_ws(&off, 4 * Q), o_touched = carve_ws(&off, touched_max), o_cnt = carve_ws(&off, 8ull * np);
    const uint64_t o_need = carve_ws(&off, 8), o_pairs = carve_ws(&off, sizeof(GvsPair) * np);
    const uint64_t p_fpairs = align_up(touched_max, 64), p_pairs = align_up(p_fpairs + sizeof(GvsPair) * np, 64);
    int rc = ensure_device(e, &e->ws, &e->ws_cap, off);
    if (!rc) rc = ensure_pinned(e, p_pairs + sizeof(GvsPair) * np);
    if (rc) return rc;
    uint8_t *ws = e->ws;
    std::vector<uint4> rows(Q, make_uint4(0xFFFFFFFFu, 0, 0, 0)), hix(Q);
    if (!keys.empty()) CU(cudaMemcpyAsync(ws + o_keys, keys.data(), keys.size(), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ws + o_off, ko.data(), 8 * (Q + 1), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ws + o_batch, qt.data(), 4 * Q, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ws + o_rows, rows.data(), 16 * Q, cudaMemcpyHostToDevice, s));
    GvsQueries gq{ws + o_keys, reinterpret_cast<const uint64_t *>(ws + o_off), reinterpret_cast<const uint32_t *>(ws + o_batch), Q,
                  reinterpret_cast<uint4 *>(ws + o_rows), reinterpret_cast<uint4 *>(ws + o_hix), reinterpret_cast<SearchState *>(ws + o_state),
                  reinterpret_cast<uint32_t *>(ws + o_node), nullptr, nullptr};
    GvsLevel L{gq, (uint32_t)((Q + 255) / 256), reinterpret_cast<GvsPair *>(ws + o_pairs), ws + o_touched, p_pairs,
               reinterpret_cast<unsigned long long *>(ws + o_need), nullptr};
    unsigned long long *d_cnt = reinterpret_cast<unsigned long long *>(ws + o_cnt);
    memcpy(e->pin + p_fpairs, pairs.data(), sizeof(GvsPair) * np);
    CU(cudaMemcpyAsync(L.d_pairs, e->pin + p_fpairs, sizeof(GvsPair) * np, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(d_cnt, 0, 8ull * np, s));
    launch_k(e, k_gvs_filter, L.grid, 256, 0, s, gq, static_cast<const GvsPair *>(L.d_pairs), d_cnt);
    std::vector<const ProbeTree *> pts(np, nullptr);
    if ((rc = gvs_level<true>(e, L, pairs, src, count, pts))) return rc;

    // ---- the bounds and the failed searches
    CU(cudaMemcpyAsync(rows.data(), ws + o_rows, 16 * Q, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(hix.data(), ws + o_hix, 16 * Q, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    for (uint64_t i = 0, q0 = 0; i < sp.size(); i++) {
        SeekPart &x = sp[i];
        const uint64_t m = x.boff.size() * x.nseek;
        x.res.assign(m, ~0ull);
        x.bad.assign(m, ~0ull);
        x.bix.assign(m, make_uint4(0, 0, 0, 0));
        for (uint64_t k = 0; k < m; k++) {
            const uint64_t q = q0 + k, rec = (uint64_t)rows[q].z | ((uint64_t)rows[q].w << 32);
            if (rows[q].y & kLookupCorrupt) {
                x.bad[k] = rec;
                x.bix[k] = hix[q];
            } else if (rows[q].x != 0xFFFFFFFFu) {
                x.res[k] = rec;
            }
        }
        q0 += m;
    }
    return DBEEL_OK;
}

// The bounds of the key ranges d < n that can hold a record (start < end; range d is kb[ko[2d] .. ko[2d + 1]) ..
// kb[ko[2d + 1] .. ko[2d + 2])) as offsets into kb and lengths: start, end, start, end, ...  Returns those ranges.
std::vector<uint32_t> range_bounds(const uint8_t *kb, const std::vector<uint64_t> &ko, uint32_t n, std::vector<uint64_t> *boff,
                                   std::vector<uint64_t> *blen) {
    std::vector<uint32_t> live;
    for (uint32_t d = 0; d < n; d++) {
        if (!key_less(kb + ko[2 * d], ko[2 * d + 1] - ko[2 * d], kb + ko[2 * d + 1], ko[2 * d + 2] - ko[2 * d + 1])) continue;
        live.push_back(d);
        for (uint32_t k = 2 * d; k < 2 * d + 2; k++) {
            boff->push_back(ko[k]);
            blen->push_back(ko[k + 1] - ko[k]);
        }
    }
    return live;
}

// The tables before the first one with no index record: a key-range read stops there with PANIC at its record 0.
uint32_t seek_tables(const dbeel_reader *r) {
    for (uint32_t t = 0; t < r->tables.size(); t++)
        if (r->tables[t]->desc.n == 0) return t;
    return (uint32_t)r->tables.size();
}

// The stop of table t's bound searches [q0, q1) of reader_seek's bad / bix: the smallest corrupt probe, PANIC when its index
// record alone shows it, as dbeel_scan on reaching the record; table -1 when none failed.
dbeel_scan_stop seek_stop(const dbeel_reader *r, uint32_t t, const std::vector<unsigned long long> &bad, const std::vector<uint4> &bix,
                          uint64_t q0, uint64_t q1) {
    uint64_t worst = q1;
    for (uint64_t q = q0; q < q1; q++)
        if (bad[q] != ~0ull && (worst == q1 || bad[q] < bad[worst])) worst = q;
    if (worst == q1) return dbeel_scan_stop{-1, DBEEL_SCAN_STOP_NONE, 0};
    const uint4 ix = bix[worst];
    const uint64_t o = (uint64_t)ix.x | ((uint64_t)ix.y << 32), dl = r->tables[t]->desc.data_len;
    const bool panic = ix.w == 0 || o > dl || ix.w > dl - o;
    return dbeel_scan_stop{(int32_t)t, panic ? DBEEL_SCAN_STOP_PANIC : DBEEL_SCAN_STOP_ERR, bad[worst]};
}

// Steps 1-2 of a key-range read on a reader (dbeel_reader_scan, dbeel_reader_get_range): the bound searches of every table
// before the first one with no index record, two per range with start < end; then the spans, merged per table, up to the
// first table whose search failed (spans->size() = that table).  *host_stop = the stop of that search or of the first empty
// table (none: table -1); a stop inside the spans lies before it in iteration order.
int reader_spans(dbeel_engine *e, dbeel_reader *r, const void *ranges, uint32_t nd, uint64_t key_bytes, const dbeel_scan_io *io,
                 std::vector<std::vector<ScanSpan>> *spans, dbeel_scan_stop *host_stop) {
    const dbeel_key_ranges *kr = static_cast<const dbeel_key_ranges *>(ranges);
    const uint8_t *kb = key_bytes ? static_cast<const uint8_t *>(kr->keys) + kr->key_offsets[0] : nullptr;
    std::vector<uint64_t> ko(2 * nd + 1);
    for (uint32_t k = 0; k <= 2 * nd; k++) ko[k] = kr->key_offsets[k] - kr->key_offsets[0];
    std::vector<uint64_t> boff, blen;
    range_bounds(kb, ko, nd, &boff, &blen);
    const uint32_t nt = (uint32_t)r->tables.size(), nseek = seek_tables(r);
    *host_stop = nseek < nt ? dbeel_scan_stop{(int32_t)nseek, DBEEL_SCAN_STOP_PANIC, 0} : dbeel_scan_stop{-1, DBEEL_SCAN_STOP_NONE, 0};
    const uint64_t nb = boff.size();
    uint32_t cutoff = nseek;
    spans->assign(nseek, {});
    if (nb && nseek) {
        std::vector<SeekPart> sp{SeekPart{r, io, nseek, kb, boff, blen, 2ull * nd, {}, {}, {}}};
        if (const int rc = reader_seek(e, sp)) return rc;
        const std::vector<unsigned long long> &res = sp[0].res, &bad = sp[0].bad;
        const std::vector<uint4> &bix = sp[0].bix;
        for (uint32_t t = 0; t < nseek; t++) {
            const dbeel_scan_stop st = seek_stop(r, t, bad, bix, nb * t, nb * (t + 1));
            if (st.table >= 0) {
                *host_stop = st;
                cutoff = t;
                break;
            }
            std::vector<ScanSpan> sp;
            for (uint64_t q = nb * t; q < nb * (t + 1); q += 2)
                if (res[q] < res[q + 1] && res[q + 1] != ~0ull) sp.push_back(ScanSpan{res[q], res[q + 1]});
            std::sort(sp.begin(), sp.end(), [](const ScanSpan &a, const ScanSpan &b) { return a.lo < b.lo; });
            for (const ScanSpan &x : sp) {
                if (!(*spans)[t].empty() && x.lo <= (*spans)[t].back().hi) (*spans)[t].back().hi = std::max((*spans)[t].back().hi, x.hi);
                else (*spans)[t].push_back(x);
            }
        }
    }
    spans->resize(cutoff);
    for (uint32_t t = 0; t < cutoff; t++)
        for (const ScanSpan &x : (*spans)[t]) e->stats.entries_in += x.hi - x.lo;
    return DBEEL_OK;
}

// Key ranges (dbeel_compact.h, dbeel_reader_scan): 1-2. reader_spans; 3. plan_scan over the spans and run_scan_plan.  The
// first stop in iteration order wins: a stop inside the spans lies before a failed search or an empty table.
int reader_scan_key(dbeel_engine *e, dbeel_reader *r, const dbeel_table *tables, const void *ranges, uint32_t nd,
                    uint64_t key_bytes, const dbeel_scan_io *io, dbeel_job_result *results, dbeel_scan_stop *stop) {
    std::vector<std::vector<ScanSpan>> spans;
    dbeel_scan_stop host_stop;
    if (const int rc = reader_spans(e, r, ranges, nd, key_bytes, io, &spans, &host_stop)) return rc;
    const int rc = plan_and_run_scan(e, tables, (uint32_t)spans.size(), DBEEL_SCAN_KEY, ranges, nd, key_bytes, io, results, stop, &spans);
    if (!rc && stop->table < 0) *stop = host_stop;
    return rc;
}

// reader_seek for many bounds, of one or many readers: each part's res / bad / bix as one reader_seek would give them.  The
// bounds are cut into seek batches whose search state (kSeekPairBytes per table and bound, plus the bound's bytes) fits
// the partition budget, each part's as its solo call cuts them, and seek batches of consecutive parts share one
// reader_seek while they fit it together (pack_batches).
int reader_seek_batched(dbeel_engine *e, std::vector<SeekPart> &parts) {
    constexpr uint64_t kSeekPairBytes = 128;
    std::vector<std::vector<uint64_t>> cost(parts.size());
    for (size_t i = 0; i < parts.size(); i++) {
        SeekPart &x = parts[i];
        const uint64_t nb = x.boff.size();
        x.res.assign(x.nseek * nb, ~0ull);
        x.bad.assign(x.nseek * nb, ~0ull);
        x.bix.assign(x.nseek * nb, make_uint4(0, 0, 0, 0));
        if (x.nseek)
            for (uint64_t j = 0; j < nb; j++) cost[i].push_back(x.blen[j] + kSeekPairBytes * x.nseek);
    }
    for (const std::vector<BatchSpan> &group : pack_batches(cost, std::vector<int32_t>(parts.size(), -1), e->partition_bytes, {})) {
        std::vector<SeekPart> sp;
        for (const BatchSpan &u : group) {
            const SeekPart &x = parts[u.batch];
            sp.push_back(SeekPart{x.r, x.io, x.nseek, x.kb, {}, {}, u.k1 - u.k0, {}, {}, {}});
            sp.back().boff.assign(x.boff.begin() + u.k0, x.boff.begin() + u.k1);
            sp.back().blen.assign(x.blen.begin() + u.k0, x.blen.begin() + u.k1);
        }
        if (const int rc = reader_seek(e, sp)) return rc;
        for (size_t i = 0; i < group.size(); i++) {
            const BatchSpan &u = group[i];
            SeekPart &x = parts[u.batch];
            const uint64_t nb = x.boff.size(), m = u.k1 - u.k0;
            for (uint64_t q = 0; q < sp[i].res.size(); q++) {
                const uint64_t at = (q / m) * nb + u.k0 + q % m;
                x.res[at] = sp[i].res[q];
                x.bad[at] = sp[i].bad[q];
                x.bix[at] = sp[i].bix[q];
            }
        }
    }
    return DBEEL_OK;
}

// ---- dbeel_reader_get_range
int discard_write(void *, uint32_t, uint32_t, uint64_t, const void *, uint64_t) { return 0; }

// Key ranges merged (dbeel_compact.h, dbeel_reader_get_range): 1-2. reader_spans; 3. plan_merge over the spans (its seek is
// reader_seek with the splitters as bounds, its key reads go through io); 4. run_scan_plan with the merge stage.  A stop --
// a failed search, an empty table, a PANIC record the planner met or a stop in a partition -- is dbeel_reader_scan's stop:
// the raw scan of the same spans is run with a discarding writer, since partitions are not in iteration order.
int reader_get_range_key(dbeel_engine *e, dbeel_reader *r, const dbeel_table *tables, const void *ranges, uint32_t nd,
                         uint64_t key_bytes, bool keep_tombstones, const dbeel_scan_io *io, dbeel_job_result *results,
                         dbeel_scan_stop *stop) {
    std::vector<std::vector<ScanSpan>> spans;
    dbeel_scan_stop host_stop;
    int rc = reader_spans(e, r, ranges, nd, key_bytes, io, &spans, &host_stop);
    if (rc) return rc;
    const uint32_t nt = (uint32_t)spans.size();
    auto raw_stop = [&]() -> int { // *stop = dbeel_reader_scan's; partitions stays the key partitions run (0: none)
        const dbeel_scan_io dio{io->read, discard_write, io->ctx};
        std::vector<dbeel_job_result> scratch(nd);
        const uint32_t parts = e->stats.partitions;
        clear_scan(results, nd, stop);
        const int src = plan_and_run_scan(e, tables, nt, DBEEL_SCAN_KEY, ranges, nd, key_bytes, &dio, scratch.data(), stop, &spans);
        if (!src && stop->table < 0) *stop = host_stop;
        e->stats.output_bytes = e->stats.entries_out = 0; // nothing that was written stands
        e->stats.partitions = parts;
        return src;
    };
    if (host_stop.table >= 0) return raw_stop();
    const MergeKeyRead read_key = [io](uint32_t t, uint64_t off, uint32_t fs, std::vector<uint8_t> *key, bool *ok) {
        constexpr uint64_t kHead = 8 + DBEEL_READER_FRAME_CAP; // most keys come with their length prefix in one read
        std::vector<uint8_t> b(std::min<uint64_t>(fs, kHead));
        *ok = false;
        if (b.size() < 8) return 0;
        if (const int krc = io->read(io->ctx, t, DBEEL_STREAM_DATA, off, b.size(), b.data())) return krc;
        uint64_t klen = 0;
        memcpy(&klen, b.data(), 8);
        if (klen > fs - 8) return 0;
        key->assign(b.begin() + 8, b.begin() + 8 + std::min<uint64_t>(klen, b.size() - 8));
        if (8 + klen > b.size()) {
            const uint64_t have = key->size();
            key->resize(klen);
            if (const int krc = io->read(io->ctx, t, DBEEL_STREAM_DATA, off + 8 + have, klen - have, key->data() + have)) return krc;
        }
        *ok = true;
        return 0;
    };
    const MergeSeek seek = [&](const std::vector<std::vector<uint8_t>> &keys, std::vector<uint64_t> *pos) {
        std::vector<uint8_t> blob;
        std::vector<uint64_t> boff, blen;
        for (const std::vector<uint8_t> &k : keys) {
            boff.push_back(blob.size());
            blen.push_back(k.size());
            blob.insert(blob.end(), k.begin(), k.end());
        }
        std::vector<SeekPart> sp{SeekPart{r, io, nt, blob.data(), boff, blen, 0, {}, {}, {}}};
        if (const int src = reader_seek_batched(e, sp)) return src;
        const std::vector<unsigned long long> &res = sp[0].res, &bad = sp[0].bad;
        pos->assign(res.size(), ~0ull);
        for (uint64_t q = 0; q < res.size(); q++) (*pos)[q] = bad[q] != ~0ull ? ~0ull : res[q];
        return 0;
    };
    const PlanTables pt = plan_tables(tables, nt, io);
    MergePlan mplan;
    rc = plan_merge(pt.dlen.data(), pt.ilen.data(), nt, e->partition_bytes, spans, pt.read_index, read_key, seek, &mplan);
    if (rc) return e->err.empty() ? fail(e, rc, "stream read callback failed (planning)") : rc;
    if (mplan.refused) { // nothing past the budget is staged: the raw scan's stop, else keys that do not ascend
        if ((rc = raw_stop()) || stop->table >= 0) return rc;
        return fail(e, DBEEL_ERR_UNSORTED_RUN, "a key interval passes the partition budget: span records do not strictly ascend");
    }
    if (mplan.plan.panic_table >= 0) return raw_stop();
    RangeMerge m{&mplan.cuts, keep_tombstones, false};
    rc = run_scan_plan(e, tables, mplan.plan, DBEEL_SCAN_KEY, ranges, nd, key_bytes, io, results, stop, &m);
    if (rc) return rc;
    if (stop->table >= 0) return raw_stop();
    if (m.unsorted) return fail(e, DBEEL_ERR_UNSORTED_RUN, "a table's span records do not strictly ascend by key");
    return DBEEL_OK;
}

// dbeel_reader_scan, or dbeel_reader_get_range when `get_range` (kind DBEEL_SCAN_KEY), on the reader's tables through its
// read callback, counted in input_bytes.  Hash ranges read every table as dbeel_scan_stream does.
int reader_range_entry(dbeel_reader *r, bool get_range, uint32_t kind, const void *ranges, uint32_t n_ranges, uint32_t flags,
                       int (*write)(void *, uint32_t, uint32_t, uint64_t, const void *, uint64_t), void *ctx,
                       dbeel_job_result *results, dbeel_scan_stop *stop) {
    dbeel_engine *e = r->e;
    if (!write) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (flags & ~DBEEL_RANGE_KEEP_TOMBSTONES) return fail(e, DBEEL_ERR_INVALID_ARG, "unknown flag");
    const std::vector<dbeel_table> tables = reader_tables(r);
    const uint32_t nt = (uint32_t)tables.size();
    uint64_t key_bytes = 0;
    if (const int arc = scan_args(e, tables.data(), nt, kind, ranges, n_ranges, results, stop, &key_bytes)) return arc;
    const Claim c(e);
    if (c.rc) return c.rc;
    clear_scan(results, n_ranges, stop);
    ReaderScanIo x;
    x.rio = &r->io;
    x.write = write;
    x.wctx = ctx;
    const dbeel_scan_io io{reader_scan_read, reader_scan_write, &x};
    if (kind == DBEEL_SCAN_HASH) return plan_and_run_scan(e, tables.data(), nt, kind, ranges, n_ranges, key_bytes, &io, results, stop, nullptr);
    const int rc = get_range ? reader_get_range_key(e, r, tables.data(), ranges, n_ranges, key_bytes,
                                                    (flags & DBEEL_RANGE_KEEP_TOMBSTONES) != 0, &io, results, stop)
                             : reader_scan_key(e, r, tables.data(), ranges, n_ranges, key_bytes, &io, results, stop);
    if (rc) {
        cudaStreamSynchronize(e->stream); // nothing of this call may touch the engine's buffers after it returns
        clear_scan(results, n_ranges, stop);
    }
    e->stats.input_bytes = x.bytes;
    return rc;
}

// ---- dbeel_reader_get_ranges / _reverse, dbeel_readers_get_ranges
// One batch of a range-read walk: its reader, the io its reads go through, its ranges (kb and ko as range_bounds takes
// them), limits, tombstone rule and direction.
struct RangeBatch {
    dbeel_reader *r;
    const dbeel_scan_io *io;
    const uint8_t *kb;
    std::vector<uint64_t> ko;
    uint32_t nq;
    const uint32_t *limits;
    bool keep_tombstones, desc;
};

// One query of a call: its batch and limit, its span [lo, hi) per searched table of its reader, the chunk width per table,
// and where its entries went.
struct LimitState {
    uint32_t batch = 0, limit = 0;
    std::vector<uint64_t> lo, hi, w;
    int32_t em = -1; // emission that holds its entries
    uint32_t at = 0; // its first entry there
};

// One merge round of a group of live queries, of any batches (range_limit.cuh): per (query, table) pair the records
// [lo, lo + w) cut at hi -- reverse: [hi - w, hi) cut at lo -- their .index slices, then the .data windows of the records
// whose index record stays inside .data, both through gvs_load with each part on its own batch's reader and io, decoded,
// merged and ranked on the device.  A (batch, table) slot is tbase[batch] + table.  A query is finished when it is
// damaged, when it has limit + 1 survivors on the complete side of its frontier, or when every pair reached its span's far
// end; the entries of the finished ones go through the split and phase 2 into emission `em` (host memory).  The pairs that
// set an unfinished query's frontier double their width; that query goes to *next.  Everything a query's row depends on is
// its own state, so its row is the same in any group.
int limit_round(dbeel_engine *e, const std::vector<RangeBatch> &bs, const std::vector<uint32_t> &tbase, const uint32_t *qs, uint32_t gq,
                std::vector<LimitState> &st, dbeel_range_row *rows, std::vector<std::vector<uint8_t>> *em, std::vector<uint32_t> *next,
                uint32_t *launches, uint64_t *gather_bytes) {
    const uint32_t nslot = tbase.back();
    cudaStream_t s = e->stream;
    int rc;
    std::vector<LimitPair> pairs;
    std::vector<uint32_t> ptab, slot_b(nslot);
    std::vector<uint64_t> pbase; // the table's record number of the pair's first staged record
    std::vector<LimitQuery> lq(gq);
    std::vector<std::vector<ByteRange>> ir(nslot);
    for (uint32_t b = 0; b + 1 < tbase.size(); b++)
        for (uint32_t k = tbase[b]; k < tbase[b + 1]; k++) slot_b[k] = b;
    uint32_t n = 0;
    for (uint32_t g = 0; g < gq; g++) {
        const LimitState &q = st[qs[g]];
        const RangeBatch &B = bs[q.batch];
        const bool desc = B.desc;
        lq[g] = LimitQuery{(uint32_t)pairs.size(), 0, n, 0, q.limit, (uint16_t)desc, (uint16_t)B.keep_tombstones};
        for (uint32_t t = 0; t < q.lo.size(); t++) {
            if (q.hi[t] <= q.lo[t]) continue;
            const uint64_t c = std::min(q.w[t], q.hi[t] - q.lo[t]), b = desc ? q.hi[t] - c : q.lo[t];
            pairs.push_back(LimitPair{n, (uint32_t)c, g, (desc ? b > q.lo[t] : b + c < q.hi[t]) ? 1u : 0u});
            ptab.push_back(t);
            pbase.push_back(b);
            ir[tbase[q.batch] + t].push_back({16 * b, 16 * (b + c)});
            n += (uint32_t)c;
        }
        lq[g].pair1 = (uint32_t)pairs.size();
        lq[g].last = n;
    }
    const uint32_t np = (uint32_t)pairs.size();
    e->stats.entries_in += n;
    // ---- the .index slices (back to host too), then the windows of the records
    std::vector<GvsStaged> ss(nslot), sw(nslot);
    std::vector<GvsPart> parts;
    auto part = [&](uint32_t k, const GvsStaged *x) {
        const RangeBatch &B = bs[slot_b[k]];
        return GvsPart{k - tbase[slot_b[k]], x, B.r, B.io};
    };
    uint64_t end = 0;
    for (uint32_t k = 0; k < nslot; k++) {
        if (ir[k].empty()) continue;
        ss[k] = gvs_stage(std::move(ir[k]), 0, end);
        end = ss[k].end;
        parts.push_back(part(k, &ss[k]));
    }
    rc = ensure_host(e, &e->ring_in, &e->ring_in_cap, end);
    if (!rc) rc = ensure_device(e, &e->stage_in, &e->stage_in_cap, end);
    if (rc) return rc;
    if ((rc = gvs_load(e, DBEEL_STREAM_INDEX, parts, e->ring_in, e->stage_in, 0, end, true, "stream read callback failed (.index, ranges)")))
        return rc;
    std::vector<uint4> rec(n);
    std::vector<uint32_t> rpair(n), pslot(np);
    std::vector<std::vector<ByteRange>> wr(nslot);
    for (uint32_t k = 0; k < np; k++) {
        const uint32_t b = st[qs[pairs[k].query]].batch, t = ptab[k], sl = pslot[k] = tbase[b] + t;
        const uint64_t dl = bs[b].r->tables[t]->desc.data_len;
        for (uint32_t j = 0; j < pairs[k].count; j++) {
            const uint8_t *ix = e->ring_in + ss[sl].at(16 * (pbase[k] + j));
            const uint64_t off = rd_le(ix, 8), fs = rd_le(ix + 12, 4);
            const bool panic = fs == 0 || off > dl || fs > dl - off; // as k_scan_classify: the index record alone shows it
            rec[pairs[k].first + j] = make_uint4(0, 0, panic ? kScanStopPanic : 0u, (uint32_t)fs);
            rpair[pairs[k].first + j] = k;
            if (!panic) wr[sl].push_back({off, off + fs});
        }
    }
    uint64_t wend = 0;
    parts.clear();
    for (uint32_t k = 0; k < nslot; k++) {
        sw[k] = gvs_stage(std::move(wr[k]), 0, wend);
        wend = sw[k].end;
        if (!sw[k].runs.empty()) parts.push_back(part(k, &sw[k]));
    }
    rc = ensure_host(e, &e->ring_out, &e->ring_out_cap, std::max<uint64_t>(wend, 256));
    if (!rc) rc = ensure_device(e, &e->stage_in2, &e->stage_in2_cap, std::max<uint64_t>(wend, 256));
    if (rc) return rc;
    if ((rc = gvs_load(e, DBEEL_STREAM_DATA, parts, e->ring_out, e->stage_in2, 0, wend, false, "stream read callback failed (.data, ranges)")))
        return rc;
    for (uint32_t k = 0; k < np; k++) {
        const uint32_t sl = pslot[k];
        for (uint32_t j = 0; j < pairs[k].count; j++) {
            uint4 &x = rec[pairs[k].first + j];
            if (x.z) continue;
            const uint64_t a = reinterpret_cast<uint64_t>(e->stage_in2 + sw[sl].at(rd_le(e->ring_in + ss[sl].at(16 * (pbase[k] + j)), 8)));
            x.x = (uint32_t)a;
            x.y = (uint32_t)(a >> 32);
        }
    }
    // ---- workspace: the round's arrays, then the split of the selected records
    const uint32_t tiles = (n + kRangeTile - 1) / kRangeTile;
    uint64_t off = 0;
    const uint64_t o_pairs = carve_ws(&off, sizeof(LimitPair) * np), o_q = carve_ws(&off, sizeof(LimitQuery) * gq);
    const uint64_t o_rec = carve_ws(&off, 16ull * n), o_rpair = carve_ws(&off, 4ull * n), o_flat = carve_ws(&off, 16ull * n);
    const uint64_t o_pfx = carve_ws(&off, 8ull * n), o_code = carve_ws(&off, 4ull * n), o_pbad = carve_ws(&off, 4ull * np);
    const uint64_t o_setter = carve_ws(&off, 4ull * np), o_front = carve_ws(&off, 4ull * gq), o_qout = carve_ws(&off, 16ull * gq);
    const uint64_t o_pre = carve_ws(&off, 4ull * (n + 1)), o_rank = carve_ws(&off, 4ull * n), o_tile = carve_ws(&off, 4ull * (tiles + 1));
    const uint64_t o_tot = carve_ws(&off, 32), o_qsel = carve_ws(&off, 4ull * gq);
    SplitLayout w = carve_split(&off, n, 1);
    if ((rc = ensure_device(e, &e->ws, &e->ws_cap, off))) return rc;
    const uint64_t pin_tot = align_up(w.header2_bytes, 64);
    if ((rc = ensure_pinned(e, pin_tot + 8ull * 4))) return rc;
    uint8_t *ws = e->ws;
    const unsigned long long tot[4] = {n, 0, 0, ~0ull}; // one segment of n records for k_range_tile_sums .. k_range_prefix
    CU(cudaMemcpyAsync(ws + o_pairs, pairs.data(), sizeof(LimitPair) * np, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ws + o_q, lq.data(), sizeof(LimitQuery) * gq, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ws + o_rec, rec.data(), 16ull * n, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ws + o_rpair, rpair.data(), 4ull * n, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ws + o_tot, tot, 32, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(ws + o_pbad, 0xFF, 4ull * np, s));
    ScanParams sp = {};
    RouteParams rp;
    Params p;
    split_bind(w, ws, &sp, &rp, &p);
    LimitParams lp{reinterpret_cast<const LimitPair *>(ws + o_pairs), reinterpret_cast<const LimitQuery *>(ws + o_q),
                   reinterpret_cast<const uint4 *>(ws + o_rec), reinterpret_cast<const uint32_t *>(ws + o_rpair), n, gq,
                   reinterpret_cast<uint4 *>(ws + o_flat), reinterpret_cast<unsigned long long *>(ws + o_pfx),
                   reinterpret_cast<uint32_t *>(ws + o_code), reinterpret_cast<uint32_t *>(ws + o_pbad), reinterpret_cast<uint32_t *>(ws + o_setter),
                   reinterpret_cast<uint32_t *>(ws + o_front), reinterpret_cast<uint4 *>(ws + o_qout), reinterpret_cast<const uint32_t *>(ws + o_pre),
                   reinterpret_cast<uint32_t *>(ws + o_pre), reinterpret_cast<uint32_t *>(ws + o_rank), reinterpret_cast<const uint32_t *>(ws + o_qsel),
                   sp.flat, sp.dest};
    RangeMergeParams mp = {};
    mp.n_ranges = 1;
    mp.totals = reinterpret_cast<unsigned long long *>(ws + o_tot);
    mp.pre = reinterpret_cast<uint32_t *>(ws + o_pre);
    mp.tile = reinterpret_cast<uint32_t *>(ws + o_tile);
    const uint32_t gn = (n + 255) / 256, gqn = (gq + 255) / 256;
    launch_k(e, k_limit_decode, gn, 256, 0, s, lp);
    launch_k(e, k_limit_query, gqn, 256, 0, s, lp);
    launch_k(e, k_limit_flag, gn, 256, 0, s, lp);
    launch_k(e, k_range_tile_sums, tiles, kRangeTile, 0, s, mp);
    launch_k(e, k_range_tile_scan, 1, kRangeTile, 0, s, mp);
    launch_k(e, k_range_prefix, tiles, kRangeTile, 0, s, mp);
    launch_k(e, k_limit_rank, std::max(gn, gqn), 256, 0, s, lp);
    *launches += 7;
    std::vector<uint4> qout(gq);
    std::vector<uint32_t> setter(np);
    CU(cudaMemcpyAsync(qout.data(), ws + o_qout, 16ull * gq, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(setter.data(), ws + o_setter, 4ull * np, cudaMemcpyDeviceToHost, s));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));
    e->stats.partitions++;

    // ---- finished queries: their rows and out slots; the others widen the pairs that hold their frontier back
    std::vector<uint32_t> qsel(gq, ~0u), done;
    uint32_t n_sel = 0;
    for (uint32_t g = 0; g < gq; g++) {
        const uint32_t qi = qs[g];
        dbeel_range_row &row = rows[qi];
        LimitState &q = st[qi];
        const uint32_t lim = q.limit;
        const uint4 o = qout[g];
        if (o.z != ~0u) {
            const uint32_t t = ptab[o.z];
            const uint64_t rec_no = pbase[o.z] + (lq[g].desc ? pairs[o.z].count - 1 - o.w : o.w); // o.w: from the chunk's fixed end
            row.flags = o.y == kLimitUnsorted ? DBEEL_RANGE_UNSORTED : DBEEL_RANGE_STOPPED;
            row.stop = dbeel_scan_stop{(int32_t)t, o.y == kLimitUnsorted ? DBEEL_SCAN_STOP_NONE : o.y, rec_no};
            continue;
        }
        bool truncated = false;
        for (uint32_t k = lq[g].pair0; k < lq[g].pair1; k++) truncated |= pairs[k].truncated != 0;
        if (o.x > lim || !truncated) {
            row.count = std::min(o.x, lim);
            row.flags = o.x > lim ? DBEEL_RANGE_MORE : 0u;
            if (row.count) {
                qsel[g] = n_sel;
                q.at = n_sel;
                q.em = (int32_t)(em->size() / 2);
                n_sel += row.count;
            }
            continue;
        }
        for (uint32_t k = lq[g].pair0; k < lq[g].pair1; k++)
            if (setter[k]) q.w[ptab[k]] *= 2;
        next->push_back(qi);
    }
    if (!n_sel) return DBEEL_OK;
    CU(cudaMemcpyAsync(ws + o_qsel, qsel.data(), 4ull * gq, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(ws + w.o_tot, 0, 8ull * 3, s));
    CU(cudaMemsetAsync(sp.stop, 0xFF, 8, s));
    launch_k(e, k_limit_select, gn, 256, 0, s, lp);
    *launches += 1;
    w.n = n_sel;
    w.n_blocks = (n_sel + kRouteThreads - 1) / kRouteThreads;
    em->emplace_back();
    em->emplace_back();
    std::vector<uint8_t> &ed = (*em)[em->size() - 2], &ei = (*em)[em->size() - 1];
    dbeel_out tmp = {};
    uint64_t items = 0, bytes = 0;
    rc = split_emit(e, w, sp, rp, p, pin_tot, false, &tmp, launches, &items, &bytes, [&](const unsigned long long *host_tot) {
        ed.resize(std::max<uint64_t>(host_tot[1], 1));
        ei.resize(16 * host_tot[0] + 16);
        tmp.data = ed.data();
        tmp.data_cap = host_tot[1];
        tmp.index = ei.data();
        tmp.index_cap = 16 * host_tot[0];
    });
    if (rc) return rc;
    *gather_bytes += e->stats.gather_bytes;
    ed.resize(bytes);
    ei.resize(16 * items);
    return DBEEL_OK;
}

// The range-read walk of dbeel_reader_get_ranges / _reverse (one batch) and dbeel_readers_get_ranges (dbeel_compact.h): the
// bound searches of every batch (reader_seek_batched over one part per batch), the spans and seek stops per query, then
// merge rounds over groups of the live queries of all batches (pack_batches: each batch's groups of about the partition
// budget as its solo call cuts them, packed whole) until every query is finished, then the rows and `out` from the
// emissions, in global query order (batch order, then query order), `first` and the .index offsets running across batches.
// Query q of batch b is row row0[b] + q.  The caller has checked the arguments, taken the engine and cleared stats, out and
// rows.
int reader_get_ranges(dbeel_engine *e, const std::vector<RangeBatch> &bs, dbeel_out *out, dbeel_range_row *rows) {
    const uint32_t nbat = (uint32_t)bs.size();
    std::vector<uint32_t> row0(nbat + 1, 0), tbase(nbat + 1, 0), nseek(nbat);
    std::vector<std::vector<uint32_t>> vq(nbat); // the queries with start < end
    std::vector<SeekPart> sp(nbat);
    for (uint32_t b = 0; b < nbat; b++) {
        const RangeBatch &B = bs[b];
        const uint32_t nt = (uint32_t)B.r->tables.size();
        nseek[b] = seek_tables(B.r);
        row0[b + 1] = row0[b] + B.nq;
        tbase[b + 1] = tbase[b] + nseek[b];
        sp[b] = SeekPart{B.r, B.io, nseek[b], B.kb, {}, {}, 0, {}, {}, {}};
        vq[b] = range_bounds(B.kb, B.ko, B.nq, &sp[b].boff, &sp[b].blen);
        const dbeel_scan_stop empty_stop{(int32_t)nseek[b], DBEEL_SCAN_STOP_PANIC, 0};
        if (nseek[b] < nt)
            for (uint32_t q = row0[b]; q < row0[b + 1]; q++) { rows[q].flags = DBEEL_RANGE_STOPPED; rows[q].stop = empty_stop; }
    }
    int rc;
    if ((rc = reader_seek_batched(e, sp))) return rc;
    CU(cudaEventRecord(e->ev[EV_START], e->stream));
    std::vector<LimitState> st(row0[nbat]);
    std::vector<uint32_t> live;
    for (uint32_t b = 0; b < nbat; b++) {
        const RangeBatch &B = bs[b];
        const uint64_t nb = sp[b].boff.size();
        for (uint32_t q = row0[b]; q < row0[b + 1]; q++) {
            st[q].batch = b;
            st[q].limit = B.limits[q - row0[b]];
        }
        if (!sp[b].nseek) continue;
        for (uint64_t j = 0; j < vq[b].size(); j++) {
            const uint32_t q = row0[b] + vq[b][j];
            LimitState &x = st[q];
            x.lo.assign(nseek[b], 0);
            x.hi.assign(nseek[b], 0);
            x.w.assign(nseek[b], (uint64_t)x.limit + 1);
            bool any = false;
            for (uint32_t t = 0; t < nseek[b]; t++) {
                const uint64_t a = t * nb + 2 * j, c = a + 1;
                const dbeel_scan_stop stop = seek_stop(B.r, t, sp[b].bad, sp[b].bix, a, c + 1);
                if (stop.table >= 0) {
                    rows[q].flags = DBEEL_RANGE_STOPPED;
                    rows[q].stop = stop;
                    any = false;
                    break;
                }
                if (sp[b].res[a] < sp[b].res[c] && sp[b].res[c] != ~0ull) {
                    x.lo[t] = sp[b].res[a];
                    x.hi[t] = sp[b].res[c];
                    any = true;
                }
            }
            if (any && !rows[q].flags) live.push_back(q);
        }
    }

    // ---- rounds: the live queries in groups of about the budget (their chunks' index records and mean entries)
    std::vector<std::vector<uint64_t>> mean(nbat);
    std::vector<int32_t> cache(nbat, -1);
    std::vector<dbeel_page_cache *> caches;
    std::vector<uint64_t> cache_bytes;
    for (uint32_t b = 0; b < nbat; b++) {
        const dbeel_reader *r = bs[b].r;
        for (uint32_t t = 0; t < nseek[b]; t++) mean[b].push_back((r->tables[t]->desc.data_len + r->tables[t]->desc.n - 1) / r->tables[t]->desc.n);
        if (!r->cache) continue;
        cache[b] = (int32_t)(std::find(caches.begin(), caches.end(), r->cache) - caches.begin());
        if (cache[b] == (int32_t)caches.size()) {
            caches.push_back(r->cache);
            cache_bytes.push_back(kPageBytes * r->cache->pc.capacity());
        }
    }
    // per staged record: its .index record, its mean entry and the round's workspace (LimitParams' arrays, the split)
    constexpr uint64_t kLimitRecordBytes = 16 + 128;
    std::vector<std::vector<uint8_t>> em; // emission k: data at 2k, index at 2k + 1
    uint32_t launches = 0;
    uint64_t gather_bytes = 0;
    while (!live.empty()) {
        std::vector<uint32_t> next;
        std::vector<std::vector<uint64_t>> cost(nbat);
        std::vector<uint32_t> live0(nbat + 1, 0); // batch b's live queries are live[live0[b] ..]
        for (const uint32_t q : live) {
            const LimitState &x = st[q];
            const uint64_t page_bytes = bs[x.batch].r->cache ? 2 * kPageBytes : 0;
            uint64_t c = 0;
            for (uint32_t t = 0; t < x.lo.size(); t++)
                if (x.hi[t] > x.lo[t]) c += std::min(x.w[t], x.hi[t] - x.lo[t]) * (kLimitRecordBytes + mean[x.batch][t]) + page_bytes;
            cost[x.batch].push_back(c);
            live0[x.batch + 1]++;
        }
        for (uint32_t b = 0; b < nbat; b++) live0[b + 1] += live0[b];
        for (const std::vector<BatchSpan> &group : pack_batches(cost, cache, e->partition_bytes, cache_bytes)) {
            std::vector<uint32_t> qs;
            for (const BatchSpan &u : group)
                qs.insert(qs.end(), live.begin() + live0[u.batch] + u.k0, live.begin() + live0[u.batch] + u.k1);
            if ((rc = limit_round(e, bs, tbase, qs.data(), (uint32_t)qs.size(), st, rows, &em, &next, &launches, &gather_bytes))) return rc;
        }
        live.swap(next);
    }

    // ---- out: every query's entries, in query order, offsets rebased
    const uint32_t nq = row0[nbat];
    uint64_t items = 0, bytes = 0;
    for (uint32_t q = 0; q < nq; q++) {
        rows[q].first = items;
        items += rows[q].count;
        if (!rows[q].count) continue;
        const uint8_t *ix = em[2 * st[q].em + 1].data() + 16ull * st[q].at;
        const uint64_t last = 16ull * (rows[q].count - 1);
        bytes += rd_le(ix + last, 8) + rd_le(ix + last + 12, 4) - rd_le(ix, 8);
    }
    if (bytes > out->data_cap || 16 * items > out->index_cap) {
        out->data_len = bytes;
        out->index_len = 16 * items;
        return fail(e, DBEEL_ERR_CAPACITY, "the entries found are larger than the output buffers (data_len / index_len: the sizes needed)");
    }
    if ((bytes && !out->data) || (items && !out->index)) return fail(e, DBEEL_ERR_INVALID_ARG, "null output buffer");
    uint8_t *od = static_cast<uint8_t *>(out->data), *oi = static_cast<uint8_t *>(out->index);
    uint64_t at = 0;
    for (uint32_t q = 0; q < nq; q++) {
        if (!rows[q].count) continue;
        const uint8_t *ix = em[2 * st[q].em + 1].data() + 16ull * st[q].at;
        const uint64_t base = rd_le(ix, 8), last = 16ull * (rows[q].count - 1);
        const uint64_t len = rd_le(ix + last, 8) + rd_le(ix + last + 12, 4) - base;
        memcpy(od + at, em[2 * st[q].em].data() + base, len);
        for (uint32_t k = 0; k < rows[q].count; k++) {
            uint8_t *dst = oi + 16ull * (rows[q].first + k);
            memcpy(dst, ix + 16ull * k, 16);
            const uint64_t o = rd_le(ix + 16ull * k, 8) - base + at;
            memcpy(dst, &o, 8);
        }
        at += len;
    }
    out->data_len = bytes;
    out->index_len = 16 * items;
    out->items_written = items;
    e->stats.kernel_launches = launches;
    e->stats.gather_bytes = gather_bytes;
    e->stats.entries_out = items;
    e->stats.output_bytes = bytes + 16 * items;
    return DBEEL_OK;
}

// The checks of one batch of key ranges with limits (dbeel_reader_get_ranges): its key offsets (ko, from 0), limits and
// flags; *total grows by its limits.
int range_batch_args(dbeel_engine *e, const dbeel_key_ranges *kr, uint32_t nq, const uint32_t *limits, uint32_t flags,
                     std::vector<uint64_t> *ko, uint64_t *total) {
    if (flags & ~DBEEL_RANGE_KEEP_TOMBSTONES) return fail(e, DBEEL_ERR_INVALID_ARG, "unknown flag");
    if (!nq) return DBEEL_OK;
    if (!kr->key_offsets || !limits) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    for (uint32_t q = 0; q < nq; q++) {
        if (limits[q] == 0 || limits[q] > DBEEL_RANGE_LIMIT_MAX) return fail(e, DBEEL_ERR_INVALID_ARG, "a limit must be 1 .. DBEEL_RANGE_LIMIT_MAX");
        *total += limits[q];
    }
    if (*total >= 0xFFFFFFF0ull) return fail(e, DBEEL_ERR_INVALID_ARG, "the limits sum to 2^32 - 16 or more");
    ko->resize(2ull * nq + 1);
    for (uint64_t k = 0; k <= 2ull * nq; k++) {
        if (k && kr->key_offsets[k] < kr->key_offsets[k - 1]) return fail(e, DBEEL_ERR_INVALID_ARG, "key_offsets must not decrease");
        (*ko)[k] = kr->key_offsets[k] - kr->key_offsets[0];
    }
    if ((*ko)[2ull * nq] && !kr->keys) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    return DBEEL_OK;
}

// Takes the engine, runs the walk over the checked batches (one ReaderScanIo each, so input_bytes counts every byte read
// through every reader's callback) and leaves rows cleared after any error other than capacity.
int ranges_entry(dbeel_engine *e, std::vector<RangeBatch> &bs, dbeel_out *out, dbeel_range_row *rows) {
    const Claim c(e);
    if (c.rc) return c.rc;
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    uint64_t nq = 0;
    for (const RangeBatch &B : bs) nq += B.nq;
    for (uint64_t q = 0; q < nq; q++) rows[q] = dbeel_range_row{0, 0, 0, dbeel_scan_stop{-1, DBEEL_SCAN_STOP_NONE, 0}};
    std::vector<ReaderScanIo> x(bs.size());
    std::vector<dbeel_scan_io> io(bs.size());
    for (size_t b = 0; b < bs.size(); b++) {
        x[b].rio = &bs[b].r->io;
        io[b] = dbeel_scan_io{reader_scan_read, nullptr, &x[b]};
        bs[b].io = &io[b];
    }
    const int rc = reader_get_ranges(e, bs, out, rows);
    if (rc && rc != DBEEL_ERR_CAPACITY) {
        cudaStreamSynchronize(e->stream); // nothing of this call may touch the engine's buffers after it returns
        for (uint64_t q = 0; q < nq; q++) rows[q] = dbeel_range_row{0, 0, 0, dbeel_scan_stop{-1, DBEEL_SCAN_STOP_NONE, 0}};
    }
    e->stats.input_bytes = 0;
    for (const ReaderScanIo &y : x) e->stats.input_bytes += y.bytes;
    return rc;
}

int reader_get_ranges_entry(dbeel_reader *r, const dbeel_key_ranges *kr, uint32_t nq, const uint32_t *limits, uint32_t flags,
                            bool desc, dbeel_out *out, dbeel_range_row *rows) {
    if (!r) return DBEEL_ERR_INVALID_ARG;
    dbeel_engine *e = r->e;
    if (!kr || !kr->key_offsets || !limits || !out || !rows) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (nq == 0) return fail(e, DBEEL_ERR_INVALID_ARG, "n_ranges must be at least 1");
    std::vector<RangeBatch> bs{RangeBatch{r, nullptr, nullptr, {}, nq, limits, (flags & DBEEL_RANGE_KEEP_TOMBSTONES) != 0, desc}};
    uint64_t total = 0;
    if (const int rc = range_batch_args(e, kr, nq, limits, flags, &bs[0].ko, &total)) return rc;
    if (bs[0].ko[2ull * nq]) bs[0].kb = static_cast<const uint8_t *>(kr->keys) + kr->key_offsets[0];
    return ranges_entry(e, bs, out, rows);
}

} // namespace

namespace dbeel {

int reader_table_create(dbeel_engine *e, const dbeel_table &t, ReaderTableRef *out) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    const Claim c(e);
    if (c.rc) return c.rc;
    // the table checks of dbeel_get_values_stream, and its filter parsed as there
    if (t.index_len % DBEEL_INDEX_ENTRY_SIZE) return fail(e, DBEEL_ERR_INVALID_ARG, "index length is not a multiple of 16");
    if (t.bloom_len && !t.bloom) return fail(e, DBEEL_ERR_INVALID_ARG, "null table buffer");
    if (t.bloom_len && (t.bloom_len < 8 + kBloomTrailer || (t.bloom_len - 8 - kBloomTrailer) % 4))
        return fail(e, DBEEL_ERR_BAD_BLOOM, "bloom file length is not 8 + 4 * words + 164");
    auto rt = std::make_shared<dbeel_reader_table>();
    rt->device = e->device;
    rt->desc = TableDesc{nullptr, t.data_len, nullptr, t.index_len / DBEEL_INDEX_ENTRY_SIZE, nullptr, 0, 0, 0, 0, {0, 0, 0, 0}};
    if (t.bloom_len) {
        const uint8_t *b = static_cast<const uint8_t *>(t.bloom);
        if (const int rc = parse_bloom(e, b, b + t.bloom_len - kBloomTrailer, t.bloom_len, &rt->desc)) return rc;
        if (cudaMalloc(reinterpret_cast<void **>(&rt->bloom_dev), t.bloom_len) != cudaSuccess) {
            cudaGetLastError();
            rt->bloom_dev = nullptr;
            return fail(e, DBEEL_ERR_NOMEM, "cudaMalloc(reader filter)");
        }
        CU(cudaMemcpy(rt->bloom_dev, b, t.bloom_len, cudaMemcpyHostToDevice));
        rt->desc.words = reinterpret_cast<const uint32_t *>(rt->bloom_dev + 8);
    }
    *out = std::move(rt);
    return DBEEL_OK;
}

int reader_open_tables(dbeel_engine *e, std::vector<ReaderTableRef> tables, const dbeel_scan_io &io, uint64_t fence_bytes,
                       std::shared_ptr<void> owner, dbeel_reader **out) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || !io.read) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (tables.size() > 65536) return fail(e, DBEEL_ERR_TOO_MANY_RUNS, "more than 65536 tables");
    const Claim c(e);
    if (c.rc) return c.rc;
    const size_t nt = tables.size();
    std::vector<uint64_t> n(nt), data_len(nt);
    std::vector<int32_t> fixed(nt);
    for (size_t i = 0; i < nt; i++) {
        n[i] = tables[i]->desc.n;
        data_len[i] = tables[i]->desc.data_len;
        fixed[i] = tables[i]->depth;
    }
    const std::vector<uint32_t> d = reader_depths(n, data_len, fixed, fence_bytes);
    for (size_t i = 0; i < nt; i++)
        if (tables[i]->depth < 0) tables[i]->depth = (int32_t)d[i];
    dbeel_reader *r = new (std::nothrow) dbeel_reader();
    if (!r) return fail(e, DBEEL_ERR_NOMEM, "reader");
    r->e = e;
    r->tables = std::move(tables);
    r->io = io;
    r->owner = std::move(owner);
    e->readers.push_back(r);
    *out = r;
    return DBEEL_OK;
}

} // namespace dbeel

// ------------------------------------------------------------------------------------ C ABI

extern "C" {

int dbeel_abi_version(void) { return DBEEL_ABI_VERSION; }

int dbeel_engine_create(int device, dbeel_engine **out) {
    if (!out) return DBEEL_ERR_INVALID_ARG;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) {
        cudaGetLastError();
        return DBEEL_ERR_NO_DEVICE;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return DBEEL_ERR_CUDA;
    if (prop.major != 9 || prop.minor != 0) return DBEEL_ERR_NO_DEVICE; // sm_90a SASS only: no fallback path
    if (cudaSetDevice(device) != cudaSuccess) return DBEEL_ERR_CUDA;
    dbeel_engine *e = new (std::nothrow) dbeel_engine();
    if (!e) return DBEEL_ERR_NOMEM;
    e->device = device;
    e->sm_count = prop.multiProcessorCount;
    if (const char *v = getenv("DBEEL_PIPELINE")) e->pipeline = atoi(v);
    if (const char *v = getenv("DBEEL_PIPELINE_MIN_KB")) e->pipeline_min_bytes = (uint64_t)(atoi(v) > 0 ? atoi(v) : 1) << 10;
    if (const char *v = getenv("DBEEL_PARTITION_KB")) e->partition_bytes = (uint64_t)(atoi(v) > 0 ? atoi(v) : 1) << 10;
    if (const char *v = getenv("DBEEL_PARTITION_TAPER")) e->partition_taper = atoi(v) != 0;
    if (const char *v = getenv("DBEEL_STREAM_RING")) e->stream_ring = std::max(2, atoi(v));
    if (const char *v = getenv("DBEEL_PARTITION_MB")) e->partition_bytes = (uint64_t)(atoi(v) > 0 ? atoi(v) : 128) << 20;
    if (cudaFuncSetAttribute(k_merge_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(2 * kMergeBufRecs * sizeof(Rec))) != cudaSuccess ||
        cudaFuncSetAttribute(k_memtable_cuts, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(12ull * kCutSlots)) != cudaSuccess) {
        dbeel_engine_destroy(e);
        return DBEEL_ERR_CUDA;
    }
    if (const char *v = getenv("DBEEL_NARROW")) e->narrow_loads = atoi(v);
    if (const char *v = getenv("DBEEL_FUSED_FINAL")) e->fused_final = atoi(v);
    if (const char *v = getenv("DBEEL_EXTRACT_PERSIST")) e->extract_persist = atoi(v);
    if (const char *v = getenv("DBEEL_PDL")) e->pdl = atoi(v);
    if (const char *v = getenv("DBEEL_STAGE_EVENTS")) e->stage_events = atoi(v);
    {
        int nb_t = 0, nb_f = 0;
        if (cudaFuncSetAttribute(k_merge_final<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFinSmem) == cudaSuccess &&
            cudaFuncSetAttribute(k_merge_final<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFinSmem) == cudaSuccess &&
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb_t, k_merge_final<true>, kFinThreads, kFinSmem) == cudaSuccess &&
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb_f, k_merge_final<false>, kFinThreads, kFinSmem) == cudaSuccess) {
            e->fin_ctas_per_sm = std::min(std::min(nb_t, nb_f), (int)DBEEL_FIN_CTAS);
        } else {
            cudaGetLastError();
            e->fin_ctas_per_sm = 0; // the five-kernel path
        }
        if (const char *v = getenv("DBEEL_FIN_CTAS_RT")) e->fin_ctas_per_sm = std::min(e->fin_ctas_per_sm, std::max(1, atoi(v)));
    }
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) { delete e; return DBEEL_ERR_CUDA; }
    for (int i = 0; i < EV_COUNT; i++)
        if (cudaEventCreate(&e->ev[i]) != cudaSuccess) { dbeel_engine_destroy(e); return DBEEL_ERR_CUDA; }
    *out = e;
    return DBEEL_OK;
}

void *dbeel_engine_stream(dbeel_engine *e) { return e ? static_cast<void *>(e->stream) : nullptr; }

void dbeel_engine_destroy(dbeel_engine *e) {
    if (!e) return;
    if (e->worker.joinable()) e->worker.join();
    cudaSetDevice(e->device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    for (dbeel_reader *r : e->readers) delete r; // the tables a tree still shares stay with the tree
    e->readers.clear();
    for (dbeel_page_cache *c : e->page_caches) delete c;
    e->page_caches.clear();
    for (int i = 0; i < EV_COUNT; i++)
        if (e->ev[i]) cudaEventDestroy(e->ev[i]);
    if (e->ws) cudaFree(e->ws);
    if (e->stage_in) cudaFree(e->stage_in);
    if (e->stage_out) cudaFree(e->stage_out);
    if (e->stage_in2) cudaFree(e->stage_in2);
    if (e->stage_out2) cudaFree(e->stage_out2);
    if (e->bloom_dev) cudaFree(e->bloom_dev);
    if (e->wal_ws) cudaFree(e->wal_ws);
    if (e->route_ws) cudaFree(e->route_ws);
    for (int i = 0; i < 2; i++) {
        if (e->ev_h2d[i]) cudaEventDestroy(e->ev_h2d[i]);
        if (e->ev_comp[i]) cudaEventDestroy(e->ev_comp[i]);
        if (e->ev_d2h[i]) cudaEventDestroy(e->ev_d2h[i]);
    }
    if (e->s_h2d) cudaStreamDestroy(e->s_h2d);
    if (e->s_d2h) cudaStreamDestroy(e->s_d2h);
    if (e->pin) cudaFreeHost(e->pin);
    if (e->ring_in) cudaFreeHost(e->ring_in);
    if (e->ring_out) cudaFreeHost(e->ring_out);
    if (e->pin_index) cudaFreeHost(e->pin_index);
    if (e->pin_bloom) cudaFreeHost(e->pin_bloom);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

// Bloom::compute_bitmap_size (bloomfilter 1.0.12): ceil(n * ln(p) / (-8 * ln2^2)) in f64
uint64_t dbeel_bloom_bitmap_bytes(uint64_t items, double fp) {
    const double ln2 = 0.693147180559945309417232121458176568; // core::f64::consts::LN_2
    return (uint64_t)ceil((double)items * log(fp) / (-8.0 * (ln2 * ln2)));
}

// Bloom::optimal_k_num: max(1, ceil(m / n * ln(2.0)))
uint32_t dbeel_bloom_k_num(uint64_t bitmap_bits, uint64_t items) {
    uint32_t k = (uint32_t)ceil((double)bitmap_bits / (double)items * log(2.0));
    return k < 1 ? 1 : k;
}

uint64_t dbeel_bloom_file_size(uint64_t items, double fp) {
    uint64_t bits = dbeel_bloom_bitmap_bytes(items, fp) * 8;
    return 8 + 4 * ((bits + 31) / 32) + 8 + 8 + 4 + 144;
}

int dbeel_compact_bound(const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts, uint64_t *data_cap,
                        uint64_t *index_cap, uint64_t *bloom_cap) {
    if (n_runs && !runs) return DBEEL_ERR_INVALID_ARG;
    dbeel_compact_opts o;
    default_opts(&o);
    if (opts) o = *opts;
    if (!(o.bloom_fp > 0.0 && o.bloom_fp < 1.0)) return DBEEL_ERR_INVALID_ARG;
    JobShape sh;
    shape_of(runs, n_runs, &o, false, &sh);
    if (data_cap) *data_cap = sh.data_total;
    if (index_cap) *index_cap = sh.n_total * 16;
    if (bloom_cap) *bloom_cap = sh.bloom_file;
    return DBEEL_OK;
}

int dbeel_compact(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts,
                  dbeel_out *out) {
    return entry(e, runs, n_runs, opts, out, false, false);
}

int dbeel_compact_stream(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts,
                         const dbeel_stream_io *io, dbeel_out *out) {
    return stream_entry(e, runs, n_runs, opts, io, out);
}

int dbeel_compact_device(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts,
                         dbeel_out *out) {
    return entry(e, runs, n_runs, opts, out, false, true);
}

int dbeel_compact_submit(dbeel_engine *e, const dbeel_run *runs, uint32_t n_runs, const dbeel_compact_opts *opts,
                         dbeel_out *out) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || (n_runs && !runs)) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    int expected = 0;
    if (!e->async_state.compare_exchange_strong(expected, 1)) return DBEEL_ERR_BUSY; // the worker owns e->err
    if (e->worker.joinable()) e->worker.join();
    e->async_runs.assign(runs, runs + n_runs); // the descriptors are copied; the buffers they point to are not
    default_opts(&e->async_opts);
    if (opts) e->async_opts = *opts;
    if (e->async_opts.bloom_seed) {
        memcpy(e->async_seed, e->async_opts.bloom_seed, 32);
        e->async_opts.bloom_seed = e->async_seed;
    }
    e->worker = std::thread([e, out]() {
        t_job_engine = e; // its Claim is not refused by its own job
        e->async_status = entry(e, e->async_runs.data(), (uint32_t)e->async_runs.size(), &e->async_opts, out, false, false);
        e->async_state.store(2, std::memory_order_release);
    });
    return DBEEL_OK;
}

int dbeel_poll(dbeel_engine *e, int *status) {
    if (!e) return 0;
    if (e->async_state.load(std::memory_order_acquire) != 2) return 0;
    if (e->worker.joinable()) e->worker.join();
    if (status) *status = e->async_status;
    e->async_state.store(0, std::memory_order_release);
    return 1;
}

int dbeel_wait(dbeel_engine *e) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (e->async_state.load(std::memory_order_acquire) == 0) return fail(e, DBEEL_ERR_INVALID_ARG, "no job in flight");
    if (e->worker.joinable()) e->worker.join();
    const int st = e->async_status;
    e->async_state.store(0, std::memory_order_release);
    return st;
}

int dbeel_flush(dbeel_engine *e, const dbeel_run *batch, dbeel_out *out) {
    return entry(e, batch, batch ? 1 : 0, nullptr, out, true, false);
}

static int flush_many_entry(dbeel_engine *e, const dbeel_run *batches, uint32_t n, dbeel_out *out, dbeel_flush_table *table,
                            bool device, bool sparse = false, uint64_t payload_bound = 0) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || !table || (n && !batches)) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    const Claim c(e);
    if (c.rc) return c.rc;
    dbeel_compact_opts o;
    default_opts(&o);
    for (uint32_t i = 0; i < n; i++) table[i] = dbeel_flush_table{0, 0, 0, 0, 0};
    JobExtra ex;
    ex.flush_table = table;
    if (sparse) { // the batches' index records point into shared .data (routed streams): no running-offset check
        ex.sparse_offsets = true;
        ex.data_bytes = payload_bound;
    }
    if (device) return run_job_device(e, batches, n, &o, true, out, &ex);
    // host buffers: stage everything down, run, bring the concatenated SSTables back
    uint64_t dsum = 0, isum = 0;
    for (uint32_t r = 0; r < n; r++) {
        if ((batches[r].data_len && !batches[r].data) || (batches[r].index_len && !batches[r].index))
            return fail(e, DBEEL_ERR_INVALID_ARG, "null batch buffer");
        dsum += batches[r].data_len;
        isum += batches[r].index_len / DBEEL_INDEX_ENTRY_SIZE * 16;
    }
    if (out->data_cap < dsum || out->index_cap < isum) return fail(e, DBEEL_ERR_CAPACITY, "output buffer too small");
    dbeel_out dout;
    const int rc = stage_outputs(e, dsum, isum, 0, &dout);
    return rc ? rc : run_job_staged(e, batches, n, &o, true, &dout, 0, out, &ex);
}

int dbeel_flush_many(dbeel_engine *e, const dbeel_run *batches, uint32_t n_batches, dbeel_out *out, dbeel_flush_table *table) {
    return flush_many_entry(e, batches, n_batches, out, table, false);
}

int dbeel_flush_many_device(dbeel_engine *e, const dbeel_run *batches, uint32_t n_batches, dbeel_out *out,
                            dbeel_flush_table *table) {
    return flush_many_entry(e, batches, n_batches, out, table, true);
}

int dbeel_flush_many_sparse_device(dbeel_engine *e, const dbeel_run *batches, uint32_t n_batches, uint64_t payload_bound,
                                   dbeel_out *out, dbeel_flush_table *table) {
    return flush_many_entry(e, batches, n_batches, out, table, true, true, payload_bound);
}

int dbeel_route_device(dbeel_engine *e, const dbeel_run *batch, const uint32_t *ring_hashes, uint32_t n_shards, void *out_index,
                       uint64_t out_index_cap, uint32_t *shard_of, void *out_key_hash64, uint64_t *counts, uint64_t *payload_bytes) {
    return route_entry(e, batch, ring_hashes, n_shards, out_index, out_index_cap, shard_of, out_key_hash64, counts, payload_bytes);
}

int dbeel_memtable_cuts_device(dbeel_engine *e, const void *key_hash64, const uint64_t *stream_starts, uint32_t n_streams,
                               uint32_t capacity, uint32_t *cuts, uint32_t *cut_starts, uint32_t max_cuts_total) {
    return cuts_entry(e, key_hash64, stream_starts, n_streams, capacity, cuts, cut_starts, max_cuts_total);
}

int dbeel_flush_device(dbeel_engine *e, const dbeel_run *batch, dbeel_out *out) {
    return entry(e, batch, batch ? 1 : 0, nullptr, out, true, true);
}

int dbeel_get_many(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys, const uint64_t *key_offsets,
                   uint64_t n_keys, uint32_t mode, dbeel_lookup_result *results) {
    return lookup_entry(e, tables, n_tables, keys, key_offsets, n_keys, mode, results, false);
}

int dbeel_get_many_device(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys,
                          const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode, dbeel_lookup_result *results) {
    return lookup_entry(e, tables, n_tables, keys, key_offsets, n_keys, mode, results, true);
}

int dbeel_get_values(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys, const uint64_t *key_offsets,
                     uint64_t n_keys, uint32_t mode, dbeel_out *out, dbeel_lookup_result *results) {
    return get_values_entry(e, tables, n_tables, keys, key_offsets, n_keys, mode, out, results, false);
}

int dbeel_get_values_device(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys,
                            const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode, dbeel_out *out, dbeel_lookup_result *results) {
    return get_values_entry(e, tables, n_tables, keys, key_offsets, n_keys, mode, out, results, true);
}

int dbeel_get_values_stream(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const void *keys,
                            const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode, const dbeel_scan_io *io,
                            dbeel_out *out, dbeel_lookup_result *results) {
    return get_values_stream_entry(e, tables, n_tables, keys, key_offsets, n_keys, mode, io, out, results);
}

int dbeel_reader_open(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, const dbeel_scan_io *io, uint64_t fence_bytes,
                      dbeel_reader **out) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out || !io || !io->read) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    if (const int arc = lookup_args(e, tables, n_tables, nullptr, 0, DBEEL_LOOKUP_REFERENCE, nullptr)) return arc;
    std::vector<ReaderTableRef> rts(n_tables);
    for (uint32_t i = 0; i < n_tables; i++)
        if (const int rc = reader_table_create(e, tables[i], &rts[i])) return rc;
    return reader_open_tables(e, std::move(rts), *io, fence_bytes, nullptr, out);
}

int dbeel_reader_get_values(dbeel_reader *r, const void *keys, const uint64_t *key_offsets, uint64_t n_keys, uint32_t mode,
                            dbeel_out *out, dbeel_lookup_result *results) {
    if (!r) return DBEEL_ERR_INVALID_ARG;
    const std::vector<dbeel_table> tables = reader_tables(r);
    return get_values_stream_entry(r->e, tables.data(), (uint32_t)tables.size(), keys, key_offsets, n_keys, mode, &r->io, out, results, r);
}

int dbeel_readers_get_values(dbeel_engine *e, const dbeel_reader_batch *batches, uint32_t n_batches, dbeel_out *out,
                             dbeel_lookup_result *results) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!batches || !out || !results) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (n_batches == 0 || n_batches > DBEEL_MAX_READER_BATCHES) return fail(e, DBEEL_ERR_INVALID_ARG, "n_batches is 0 or above DBEEL_MAX_READER_BATCHES");
    uint64_t n_keys = 0;
    for (uint32_t b = 0; b < n_batches; b++) {
        const dbeel_reader_batch &x = batches[b];
        if (!x.reader) return fail(e, DBEEL_ERR_INVALID_ARG, "null reader");
        if (x.reader->e != e) return fail(e, DBEEL_ERR_INVALID_ARG, "a reader of another engine");
        if (x.mode > DBEEL_LOOKUP_EXACT) return fail(e, DBEEL_ERR_INVALID_ARG, "unknown lookup mode");
        if (x.reserved) return fail(e, DBEEL_ERR_INVALID_ARG, "reserved is not 0");
        if (!x.key_offsets) return fail(e, DBEEL_ERR_INVALID_ARG, "null key_offsets");
        if (x.n_keys >= 0xFFFFFFF0ull - n_keys) return fail(e, DBEEL_ERR_INVALID_ARG, "2^32 - 16 keys or more");
        if (!x.keys && x.key_offsets[x.n_keys] > x.key_offsets[0]) return fail(e, DBEEL_ERR_INVALID_ARG, "null keys with key bytes");
        n_keys += x.n_keys;
    }
    const Claim c(e);
    if (c.rc) return c.rc;
    out->data_len = out->index_len = out->bloom_len = out->items_written = 0;
    std::vector<GvsBatch> bs(n_batches);
    for (uint32_t b = 0; b < n_batches; b++) {
        const dbeel_reader_batch &x = batches[b];
        GvsBatch &B = bs[b];
        B.r = x.reader;
        B.io = &x.reader->io;
        B.keys = static_cast<const uint8_t *>(x.keys);
        B.key_off = x.key_offsets;
        B.n_keys = x.n_keys;
        B.mode = x.mode;
        for (uint64_t q = 0; q < x.n_keys; q++) B.max_klen = std::max(B.max_klen, x.key_offsets[q + 1] - x.key_offsets[q]);
        for (const ReaderTableRef &t : x.reader->tables) B.td.push_back(t->desc);
    }
    return gvs_walk(e, bs, out, results);
}

int dbeel_reader_scan(dbeel_reader *r, uint32_t kind, const void *ranges, uint32_t n_ranges,
                      int (*write)(void *ctx, uint32_t dest, uint32_t kind, uint64_t offset, const void *src, uint64_t len),
                      void *ctx, dbeel_job_result *results, dbeel_scan_stop *stop) {
    if (!r) return DBEEL_ERR_INVALID_ARG;
    return reader_range_entry(r, false, kind, ranges, n_ranges, 0, write, ctx, results, stop);
}

void dbeel_reader_close(dbeel_reader *r) {
    if (!r) return;
    auto &v = r->e->readers;
    v.erase(std::remove(v.begin(), v.end(), r), v.end());
    cudaSetDevice(r->e->device);
    delete r;
}

int dbeel_reader_get_range(dbeel_reader *r, const dbeel_key_ranges *ranges, uint32_t n_ranges, uint32_t flags,
                           int (*write)(void *ctx, uint32_t dest, uint32_t kind, uint64_t offset, const void *src, uint64_t len),
                           void *ctx, dbeel_job_result *results, dbeel_scan_stop *stop) {
    if (!r) return DBEEL_ERR_INVALID_ARG;
    return reader_range_entry(r, true, DBEEL_SCAN_KEY, ranges, n_ranges, flags, write, ctx, results, stop);
}

int dbeel_reader_get_ranges(dbeel_reader *r, const dbeel_key_ranges *ranges, uint32_t n_ranges, const uint32_t *limits,
                            uint32_t flags, dbeel_out *out, dbeel_range_row *rows) {
    if (!r) return DBEEL_ERR_INVALID_ARG;
    return reader_get_ranges_entry(r, ranges, n_ranges, limits, flags, false, out, rows);
}

int dbeel_reader_get_ranges_reverse(dbeel_reader *r, const dbeel_key_ranges *ranges, uint32_t n_ranges, const uint32_t *limits,
                                    uint32_t flags, dbeel_out *out, dbeel_range_row *rows) {
    if (!r) return DBEEL_ERR_INVALID_ARG;
    return reader_get_ranges_entry(r, ranges, n_ranges, limits, flags, true, out, rows);
}

int dbeel_readers_get_ranges(dbeel_engine *e, const dbeel_range_batch *batches, uint32_t n_batches, dbeel_out *out,
                             dbeel_range_row *rows) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!batches || !out || !rows) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    if (n_batches == 0 || n_batches > DBEEL_MAX_READER_BATCHES) return fail(e, DBEEL_ERR_INVALID_ARG, "n_batches is 0 or above DBEEL_MAX_READER_BATCHES");
    std::vector<RangeBatch> bs(n_batches);
    uint64_t total = 0;
    for (uint32_t b = 0; b < n_batches; b++) {
        const dbeel_range_batch &x = batches[b];
        if (!x.reader) return fail(e, DBEEL_ERR_INVALID_ARG, "null reader");
        if (x.reader->e != e) return fail(e, DBEEL_ERR_INVALID_ARG, "a reader of another engine");
        if (x.reverse > 1) return fail(e, DBEEL_ERR_INVALID_ARG, "reverse is not 0 or 1");
        if (x.reserved) return fail(e, DBEEL_ERR_INVALID_ARG, "reserved is not 0");
        bs[b] = RangeBatch{x.reader, nullptr, nullptr, {}, x.n_ranges, x.limits, (x.flags & DBEEL_RANGE_KEEP_TOMBSTONES) != 0, x.reverse != 0};
        if (const int rc = range_batch_args(e, &x.ranges, x.n_ranges, x.limits, x.flags, &bs[b].ko, &total)) return rc;
        if (x.n_ranges && bs[b].ko[2ull * x.n_ranges]) bs[b].kb = static_cast<const uint8_t *>(x.ranges.keys) + x.ranges.key_offsets[0];
    }
    return ranges_entry(e, bs, out, rows);
}

int dbeel_page_cache_create(dbeel_engine *e, uint64_t bytes, dbeel_page_cache **out) {
    if (!e) return DBEEL_ERR_INVALID_ARG;
    if (!out) return fail(e, DBEEL_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    const uint64_t slots = bytes / kPageBytes;
    if (slots == 0) return fail(e, DBEEL_ERR_INVALID_ARG, "a page cache needs at least one 4096-byte page");
    if (slots > 0xFFFFFFFFull) return fail(e, DBEEL_ERR_INVALID_ARG, "a page cache holds at most 2^32 - 1 pages");
    const Claim claim(e);
    if (claim.rc) return claim.rc;
    uint8_t *pool = nullptr;
    cudaError_t ce = cudaMalloc(reinterpret_cast<void **>(&pool), slots * kPageBytes);
    if (ce != cudaSuccess) { cudaGetLastError(); return fail(e, DBEEL_ERR_NOMEM, "cudaMalloc(page cache)", ce); }
    dbeel_page_cache *c = new (std::nothrow) dbeel_page_cache(slots);
    if (!c) { cudaFree(pool); return fail(e, DBEEL_ERR_NOMEM, "page cache"); }
    c->e = e;
    c->pool = pool;
    e->page_caches.push_back(c);
    *out = c;
    return DBEEL_OK;
}

void dbeel_page_cache_destroy(dbeel_page_cache *c) {
    if (!c) return;
    dbeel_engine *e = c->e;
    for (dbeel_reader *r : e->readers)
        if (r->cache == c) r->cache = nullptr;
    auto &v = e->page_caches;
    v.erase(std::remove(v.begin(), v.end(), c), v.end());
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream); // copies still reading its slots
    delete c;
}

int dbeel_reader_attach_page_cache(dbeel_reader *r, dbeel_page_cache *c) {
    if (!r) return DBEEL_ERR_INVALID_ARG;
    dbeel_engine *e = r->e;
    if (c && c->e != e) return fail(e, DBEEL_ERR_INVALID_ARG, "the page cache belongs to another engine");
    const Claim claim(e);
    if (claim.rc) return claim.rc;
    r->cache = c;
    return DBEEL_OK;
}

int dbeel_page_cache_stats(const dbeel_page_cache *c, struct dbeel_page_cache_stats *out) {
    if (!c || !out) return DBEEL_ERR_INVALID_ARG;
    const Claim claim(c->e);
    if (claim.rc) return claim.rc;
    out->capacity_pages = c->pc.capacity();
    out->resident_pages = c->pc.resident();
    out->hits = c->pc.hits;
    out->misses = c->pc.misses;
    out->evictions = c->pc.evictions;
    return DBEEL_OK;
}

int dbeel_scan_bound(const dbeel_table *tables, uint32_t n_tables, uint64_t *data_cap, uint64_t *index_cap) {
    if (n_tables && !tables) return DBEEL_ERR_INVALID_ARG;
    uint64_t d = 0, i = 0;
    for (uint32_t t = 0; t < n_tables; t++) { d += tables[t].data_len; i += tables[t].index_len; }
    if (data_cap) *data_cap = d;
    if (index_cap) *index_cap = i;
    return DBEEL_OK;
}

int dbeel_scan(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges, uint32_t n_ranges,
               dbeel_out *out, dbeel_job_result *results, dbeel_scan_stop *stop) {
    return scan_entry(e, tables, n_tables, kind, ranges, n_ranges, out, results, stop, false);
}

int dbeel_scan_device(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges,
                      uint32_t n_ranges, dbeel_out *out, dbeel_job_result *results, dbeel_scan_stop *stop) {
    return scan_entry(e, tables, n_tables, kind, ranges, n_ranges, out, results, stop, true);
}

int dbeel_scan_stream(dbeel_engine *e, const dbeel_table *tables, uint32_t n_tables, uint32_t kind, const void *ranges,
                      uint32_t n_ranges, const dbeel_scan_io *io, dbeel_job_result *results, dbeel_scan_stop *stop) {
    return scan_stream_entry(e, tables, n_tables, kind, ranges, n_ranges, io, results, stop);
}

int dbeel_compact_many_bound(const dbeel_job *jobs, uint32_t n_jobs, uint64_t bloom_min_size, double bloom_fp, uint64_t *data_cap,
                             uint64_t *index_cap, uint64_t *bloom_cap) {
    if (n_jobs && !jobs) return DBEEL_ERR_INVALID_ARG;
    JobShapes js;
    int rc = job_shapes(nullptr, jobs, n_jobs, bloom_min_size, bloom_fp, &js);
    if (rc) return rc;
    if (data_cap) *data_cap = js.data;
    if (index_cap) *index_cap = js.index;
    if (bloom_cap) *bloom_cap = js.bloom;
    return DBEEL_OK;
}

int dbeel_compact_many(dbeel_engine *e, const dbeel_job *jobs, uint32_t n_jobs, uint64_t bloom_min_size, double bloom_fp,
                       dbeel_out *out, dbeel_job_result *results) {
    return compact_many_entry(e, jobs, n_jobs, bloom_min_size, bloom_fp, out, results, false);
}

int dbeel_compact_many_device(dbeel_engine *e, const dbeel_job *jobs, uint32_t n_jobs, uint64_t bloom_min_size, double bloom_fp,
                              dbeel_out *out, dbeel_job_result *results) {
    return compact_many_entry(e, jobs, n_jobs, bloom_min_size, bloom_fp, out, results, true);
}

int dbeel_wal_flush(dbeel_engine *e, const void *wal, uint64_t wal_len, uint32_t capacity, dbeel_out *out) {
    return wal_flush_entry(e, wal, wal_len, capacity, out, false);
}

int dbeel_wal_flush_device(dbeel_engine *e, const void *wal, uint64_t wal_len, uint32_t capacity, dbeel_out *out) {
    return wal_flush_entry(e, wal, wal_len, capacity, out, true);
}

void *dbeel_host_alloc(uint64_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

void dbeel_host_free(void *p) {
    if (p) cudaFreeHost(p);
}

// Stats and the error text of an asynchronous job belong to its worker thread until dbeel_poll / dbeel_wait has joined it.
int dbeel_last_stats(const dbeel_engine *e, dbeel_stats *out) {
    if (!e || !out) return DBEEL_ERR_INVALID_ARG;
    if (e->async_state.load(std::memory_order_acquire) != 0) return DBEEL_ERR_BUSY;
    *out = e->stats;
    return DBEEL_OK;
}

const char *dbeel_last_error(const dbeel_engine *e) {
    if (!e) return "null engine";
    if (e->async_state.load(std::memory_order_acquire) != 0) return "an asynchronous job is in flight";
    return e->err.c_str();
}

const char *dbeel_strerror(int code) {
    switch (code) {
    case DBEEL_OK: return "ok";
    case DBEEL_ERR_INVALID_ARG: return "invalid argument";
    case DBEEL_ERR_CAPACITY: return "output buffer too small";
    case DBEEL_ERR_ITEM_TOO_LARGE: return "item too large";
    case DBEEL_ERR_CUDA: return "CUDA error";
    case DBEEL_ERR_NOMEM: return "out of memory";
    case DBEEL_ERR_TOO_MANY_RUNS: return "too many runs";
    case DBEEL_ERR_TOO_MANY_ENTRIES: return "too many entries";
    case DBEEL_ERR_UNSORTED_RUN: return "input run not strictly ascending";
    case DBEEL_ERR_NO_DEVICE: return "no sm_90 CUDA device";
    case DBEEL_ERR_BUSY: return "engine busy";
    case DBEEL_ERR_BAD_BLOOM: return "malformed .bloom file";
    case DBEEL_ERR_TREE_FULL: return "memtable capacity reached";
    default: return "unknown error";
    }
}

} // extern "C"
