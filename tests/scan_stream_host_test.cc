// scan_stream_host_test.cc -- the host side of dbeel_scan_stream without a GPU.
//
//   pump              StreamPump with per-destination output pieces (the scan's writer side): every byte of every
//                     destination's two files arrives exactly once at its offset, pieces longer than kPiece included;
//                     an error from either callback stops the pump and the first code wins.
//   pump-far          the same writer loop with file offsets past 2^32, for the scan's pieces and the compaction's OutPart.
//   plan B1 B2 ...    reads a tree from stdin ("n_tables", then per table "data_len index_path"), plans it with
//                     dbeel_b200/csrc/host/scan_plan.h at every budget and prints the plan (tests/test_scan_stream_host.py
//                     checks it against the records and the scan oracle).
//
//   g++ -O2 -std=c++17 -pthread tests/scan_stream_host_test.cc -o /tmp/scan_stream_host_test
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <random>
#include <string>

#include "../dbeel_b200/csrc/host/scan_plan.h"
#include "../dbeel_b200/csrc/host/stream_pump.h"

using dbeel::StreamPump;

namespace {

struct Files {
    std::vector<uint8_t> input;                  // one input "table"
    std::vector<std::vector<uint8_t>> out[3];    // [kind][dest]
    std::vector<std::vector<uint8_t>> hits[3];
    std::atomic<int> reads{0}, writes{0};
    int fail_read_at = -1, fail_write_at = -1;
    std::mutex mu;
};

int rd(void *ctx, uint32_t, uint32_t, uint64_t off, uint64_t len, void *dst) {
    Files *f = static_cast<Files *>(ctx);
    const int k = f->reads.fetch_add(1);
    if (k == f->fail_read_at) return 77;
    if (off + len > f->input.size()) return 78;
    if ((k & 7) == 0) std::this_thread::sleep_for(std::chrono::microseconds(200));
    memcpy(dst, f->input.data() + off, len);
    return 0;
}

int wr(void *ctx, uint32_t dest, uint32_t kind, uint64_t off, const void *src, uint64_t len) {
    Files *f = static_cast<Files *>(ctx);
    const int k = f->writes.fetch_add(1);
    if (k == f->fail_write_at) return 88;
    if (kind != DBEEL_STREAM_DATA && kind != DBEEL_STREAM_INDEX) return 89;
    std::vector<uint8_t> &dst = f->out[kind][dest];
    if (off + len > dst.size()) return 90;
    if ((k & 3) == 0) std::this_thread::sleep_for(std::chrono::microseconds(100));
    memcpy(dst.data() + off, src, len);
    std::lock_guard<std::mutex> lk(f->mu);
    for (uint64_t i = 0; i < len; i++) f->hits[kind][dest][off + i]++;
    return 0;
}

// np partitions, nd destinations: partition c's piece of (dest, kind) is a random length (some empty, some > kPiece); the
// "engine" reads partition c's input slice, then publishes the pieces, which point into a per-partition buffer filled
// from a seeded pattern.  Returns 0, or the pump's error code.
int pump_scenario(uint32_t np, uint32_t nd, uint32_t ring, int threads, uint64_t max_piece, unsigned seed, int fail_read_at, int fail_write_at) {
    std::mt19937_64 rng(seed);
    Files f;
    f.fail_read_at = fail_read_at;
    f.fail_write_at = fail_write_at;
    f.input.resize(4096ull * np);
    std::vector<std::vector<std::array<uint64_t, 3>>> len(np, std::vector<std::array<uint64_t, 3>>(nd)); // [c][d][kind]
    std::vector<std::array<uint64_t, 3>> total(nd, {0, 0, 0});
    for (uint32_t c = 0; c < np; c++)
        for (uint32_t d = 0; d < nd; d++)
            for (uint32_t k = 1; k <= 2; k++) {
                const uint64_t n = rng() % 4 == 0 ? 0 : (rng() % 50 == 0 ? StreamPump::kPiece + rng() % max_piece : rng() % max_piece);
                len[c][d][k] = n;
                total[d][k] += n;
            }
    for (uint32_t k = 1; k <= 2; k++) {
        f.out[k].resize(nd);
        f.hits[k].resize(nd);
        for (uint32_t d = 0; d < nd; d++) { f.out[k][d].assign(total[d][k], 0); f.hits[k][d].assign(total[d][k], 0); }
    }
    auto byte_of = [](uint32_t d, uint32_t k, uint64_t i) { return (uint8_t)(d * 31 + k * 7 + i * 13 + (i >> 9)); };
    std::vector<std::vector<uint8_t>> bufs(np);
    std::vector<uint8_t> slots((uint64_t)ring * 4096);
    dbeel_scan_io io{rd, wr, &f};
    StreamPump pump(&io, np, ring, threads, [](uint32_t) {});
    for (uint32_t c = 0; c < np; c++) pump.add_read(c, 0, DBEEL_STREAM_DATA, 4096ull * c, 4096, slots.data() + (c % ring) * 4096ull);
    pump.start();
    std::vector<std::array<uint64_t, 3>> at(nd, {0, 0, 0});
    int rc = 0;
    for (uint32_t c = 0; c < np && !rc; c++) {
        rc = pump.wait_reads(c);
        if (rc) break;
        if (memcmp(slots.data() + (c % ring) * 4096ull, f.input.data() + 4096ull * c, 4096) != 0) { fprintf(stderr, "slot %u refilled early\n", c); return -1; }
        pump.release_input(c);
        rc = pump.wait_out_slot(c);
        if (rc) break;
        uint64_t sz = 0;
        for (uint32_t d = 0; d < nd; d++) sz += len[c][d][1] + len[c][d][2];
        bufs[c].resize(sz);
        std::vector<StreamPump::OutPiece> ps;
        uint64_t pos = 0;
        for (uint32_t d = 0; d < nd; d++)
            for (uint32_t k = 1; k <= 2; k++) {
                for (uint64_t i = 0; i < len[c][d][k]; i++) bufs[c][pos + i] = byte_of(d, k, at[d][k] + i);
                ps.push_back({d, k, at[d][k], bufs[c].data() + pos, len[c][d][k]});
                at[d][k] += len[c][d][k];
                pos += len[c][d][k];
            }
        pump.publish_pieces(c, std::move(ps));
    }
    if (rc) pump.abort(rc);
    const int frc = rc ? rc : pump.finish();
    if (frc) return frc;
    for (uint32_t d = 0; d < nd; d++)
        for (uint32_t k = 1; k <= 2; k++)
            for (uint64_t i = 0; i < total[d][k]; i++)
                if (f.out[k][d][i] != byte_of(d, k, i) || f.hits[k][d][i] != 1) {
                    fprintf(stderr, "dest %u kind %u byte %llu wrong (hits %u)\n", d, k, (unsigned long long)i, f.hits[k][d][i]);
                    return -2;
                }
    return 0;
}

int run_pump() {
    int bad = 0;
    unsigned seed = 1;
    for (uint32_t np : {1u, 2u, 5u, 17u})
        for (uint32_t nd : {1u, 3u, 40u})
            for (uint32_t ring : {2u, 3u})
                for (int threads : {1, 4, 8}) {
                    const int rc = pump_scenario(np, nd, ring, threads, 2000, seed++, -1, -1);
                    if (rc) { fprintf(stderr, "np=%u nd=%u ring=%u threads=%d -> %d\n", np, nd, ring, threads, rc); bad++; }
                }
    for (int at : {0, 2, 9}) {
        int rc = pump_scenario(12, 6, 3, 4, 2000, 500 + at, at, -1);
        if (rc != 77) { fprintf(stderr, "read failure at %d -> %d (want 77)\n", at, rc); bad++; }
    }
    for (int at : {0, 5, 60}) {
        int rc = pump_scenario(12, 6, 3, 4, 2000, 600 + at, -1, at);
        if (rc != 88) { fprintf(stderr, "write failure at %d -> %d (want 88)\n", at, rc); bad++; }
        // both fail: whichever callback failed first, its code is the one returned
        rc = pump_scenario(12, 6, 3, 4, 2000, 700 + at, 7, at);
        if (rc != 77 && rc != 88) { fprintf(stderr, "both failures at %d -> %d\n", at, rc); bad++; }
    }
    printf(bad ? "FAILED %d\n" : "ok\n", bad);
    return bad ? 1 : 0;
}

// Output pieces at file offsets past 2^32 (a destination file larger than 4 GiB): destination d's files start a little
// over one kPiece below (d + 1) << 32, so pieces, and the kPiece-sized calls a long piece is split into, cross 2^32 and
// 2^33.  No file is kept: the write callback checks every byte against a pattern of its absolute 64-bit offset (a write
// at an offset truncated to 32 bits fails it) and records the range it covered.
uint8_t far_byte(uint32_t d, uint32_t k, uint64_t off) {
    return (uint8_t)((off >> 32) * 37 + off * 13 + (off >> 11) + d * 31 + k * 7);
}

struct FarFiles {
    std::mutex mu;
    std::vector<std::array<uint64_t, 4>> calls; // dest, kind, offset, len
    int bad = 0;
};

int far_check(FarFiles *f, uint32_t dest, uint32_t kind, uint64_t off, const void *src, uint64_t len) {
    const uint8_t *p = static_cast<const uint8_t *>(src);
    for (uint64_t i = 0; i < len; i++)
        if (p[i] != far_byte(dest, kind, off + i)) return 91;
    std::lock_guard<std::mutex> lk(f->mu);
    f->calls.push_back({dest, kind, off, len});
    return 0;
}

int wr_far(void *ctx, uint32_t dest, uint32_t kind, uint64_t off, const void *src, uint64_t len) {
    return far_check(static_cast<FarFiles *>(ctx), dest, kind, off, src, len);
}

int wr_far_compact(void *ctx, uint32_t kind, uint64_t off, const void *src, uint64_t len) {
    return far_check(static_cast<FarFiles *>(ctx), 0, kind, off, src, len);
}

int rd_none(void *, uint32_t, uint32_t, uint64_t, uint64_t, void *) { return 0; }

// The calls of every (dest, kind) tile [start, start + total) exactly once; returns the number of calls crossing a
// multiple of 2^32, or -1.
long far_coverage(FarFiles &f, uint32_t nd, const std::vector<std::array<uint64_t, 3>> &start,
                  const std::vector<std::array<uint64_t, 3>> &total) {
    long crossing = 0;
    for (uint32_t d = 0; d < nd; d++)
        for (uint32_t k = 1; k <= 2; k++) {
            std::vector<std::pair<uint64_t, uint64_t>> r;
            for (const auto &c : f.calls)
                if (c[0] == d && c[1] == k) r.push_back({c[2], c[3]});
            std::sort(r.begin(), r.end());
            uint64_t at = start[d][k];
            for (const auto &x : r) {
                if (x.first != at) {
                    fprintf(stderr, "dest %u kind %u: call at %llu, expected %llu\n", d, k, (unsigned long long)x.first,
                            (unsigned long long)at);
                    return -1;
                }
                if (x.first >> 32 != (x.first + x.second - 1) >> 32) crossing++;
                at += x.second;
            }
            if (at != start[d][k] + total[d][k]) {
                fprintf(stderr, "dest %u kind %u: ends at %llu, expected %llu\n", d, k, (unsigned long long)at,
                        (unsigned long long)(start[d][k] + total[d][k]));
                return -1;
            }
        }
    return crossing;
}

int pump_far_scenario(uint32_t np, uint32_t nd, uint32_t ring, int threads, unsigned seed, bool compact) {
    std::mt19937_64 rng(seed);
    FarFiles f;
    const uint64_t P = StreamPump::kPiece;
    std::vector<std::array<uint64_t, 3>> start(nd), total(nd, {0, 0, 0}), at(nd);
    for (uint32_t d = 0; d < nd; d++)
        for (uint32_t k = 1; k <= 2; k++) start[d][k] = at[d][k] = ((uint64_t)(d + 1) << 32) - P - P / 2 - 5 - 11 * k;
    std::vector<std::vector<uint8_t>> bufs(np);
    dbeel_scan_io sio{rd_none, wr_far, &f};
    dbeel_stream_io cio{rd_none, wr_far_compact, &f};
    std::unique_ptr<StreamPump> pump(compact ? new StreamPump(&cio, np, ring, threads, [](uint32_t) {})
                                             : new StreamPump(&sio, np, ring, threads, [](uint32_t) {}));
    pump->start();
    for (uint32_t c = 0; c < np; c++) {
        if (pump->wait_out_slot(c)) return -3;
        uint64_t len[64][3] = {};
        uint64_t sz = 0;
        for (uint32_t d = 0; d < nd; d++)
            for (uint32_t k = 1; k <= 2; k++) {
                // partition 0's piece alone runs past (d + 1) << 32; later ones: empty, short or longer than kPiece
                len[d][k] = c == 0 ? P + P / 2 + 5 + 11 * k + 1 + rng() % P
                                   : rng() % 5 == 0 ? 0 : (rng() % 3 == 0 ? P + rng() % (P + P / 2) : 1 + rng() % (P / 3));
                sz += len[d][k];
            }
        bufs[c].resize(sz);
        std::vector<StreamPump::OutPiece> ps;
        uint64_t pos = 0;
        for (uint32_t d = 0; d < nd; d++)
            for (uint32_t k = 1; k <= 2; k++) {
                for (uint64_t i = 0; i < len[d][k]; i++) bufs[c][pos + i] = far_byte(d, k, at[d][k] + i);
                ps.push_back({d, k, at[d][k], bufs[c].data() + pos, len[d][k]});
                at[d][k] += len[d][k];
                total[d][k] += len[d][k];
                pos += len[d][k];
            }
        if (compact) {
            StreamPump::OutPart o;
            o.data = ps[0].src, o.data_len = ps[0].len, o.data_off = ps[0].off;
            o.index = ps[1].src, o.index_len = ps[1].len, o.index_off = ps[1].off;
            pump->publish_out(c, o);
        } else {
            pump->publish_pieces(c, std::move(ps));
        }
    }
    const int rc = pump->finish();
    if (rc) return rc;
    const long crossing = far_coverage(f, nd, start, total);
    if (crossing < 0) return -2;
    for (uint32_t d = 0; d < nd; d++)
        for (uint32_t k = 1; k <= 2; k++)
            if (start[d][k] + total[d][k] <= ((uint64_t)(d + 1) << 32)) {
                fprintf(stderr, "dest %u kind %u never reaches %u << 32\n", d, k, d + 1);
                return -4;
            }
    return crossing > 0 ? 0 : -5;
}

int run_pump_far() {
    int bad = 0;
    unsigned seed = 40;
    for (bool compact : {false, true})
        for (uint32_t ring : {2u, 3u})
            for (int threads : {1, 4}) {
                const uint32_t nd = compact ? 1 : 3;
                const int rc = pump_far_scenario(5, nd, ring, threads, seed++, compact);
                if (rc) { fprintf(stderr, "%s ring=%u threads=%d -> %d\n", compact ? "OutPart" : "pieces", ring, threads, rc); bad++; }
            }
    printf(bad ? "FAILED %d\n" : "ok\n", bad);
    return bad ? 1 : 0;
}

int run_plan(int argc, char **argv) {
    uint32_t n = 0;
    if (scanf("%u", &n) != 1) return 2;
    std::vector<uint64_t> dlen(n), ilen(n);
    std::vector<std::vector<uint8_t>> index(n);
    for (uint32_t t = 0; t < n; t++) {
        unsigned long long dl;
        char path[4096];
        if (scanf("%llu %4095s", &dl, path) != 2) return 2;
        dlen[t] = dl;
        FILE *fp = fopen(path, "rb");
        if (!fp) return 3;
        uint8_t b[65536];
        size_t r;
        while ((r = fread(b, 1, sizeof b, fp)) > 0) index[t].insert(index[t].end(), b, b + r);
        fclose(fp);
        ilen[t] = index[t].size();
    }
    uint64_t max_read = 0;
    auto read = [&](uint32_t t, uint64_t off, uint64_t len, void *dst) {
        if (off + len > index[t].size()) return 5;
        if (len > max_read) max_read = len;
        memcpy(dst, index[t].data() + off, len);
        return 0;
    };
    for (int a = 2; a < argc; a++) {
        const uint64_t budget = strtoull(argv[a], nullptr, 10);
        dbeel::ScanPlan plan;
        const int rc = dbeel::plan_scan(dlen.data(), ilen.data(), n, budget, read, &plan);
        if (rc) return 4;
        printf("budget %llu parts %zu panic %d %llu\n", (unsigned long long)budget, plan.parts.size(), plan.panic_table,
               (unsigned long long)plan.panic_record);
        for (const dbeel::ScanPart &p : plan.parts) {
            printf("part %llu %llu %u\n", (unsigned long long)p.n_rec, (unsigned long long)p.data_bound, p.n_slices);
            for (uint32_t k = 0; k < p.n_slices; k++) {
                const dbeel::ScanSlice &s = plan.slices[p.first_slice + k];
                printf("slice %u %llu %llu %llu %llu\n", s.table, (unsigned long long)s.rec_lo, (unsigned long long)s.rec_hi,
                       (unsigned long long)s.win_lo, (unsigned long long)s.win_hi);
            }
        }
    }
    printf("max_read %llu\n", (unsigned long long)max_read);
    return 0;
}

} // namespace

int main(int argc, char **argv) {
    if (argc >= 2 && !strcmp(argv[1], "pump")) return run_pump();
    if (argc >= 2 && !strcmp(argv[1], "pump-far")) return run_pump_far();
    if (argc >= 3 && !strcmp(argv[1], "plan")) return run_plan(argc, argv);
    fprintf(stderr, "usage: %s pump | pump-far | plan BUDGET... < tree\n", argv[0]);
    return 2;
}
