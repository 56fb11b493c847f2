// stream_pump.h -- the threads between a file (the caller's read / write callbacks) and the pinned rings of the streaming
// host path (dbeel_compact_stream, row N3: the storage edge).  Plain C++: no CUDA in here, so the flow control is
// exercised on a box without a GPU (tests/stream_pump_test.cc); the engine supplies "wait until partition c's D2H has
// landed" as a callable.
//
// The pipeline of dbeel_compact.cu walks the key-range partitions of a compaction in order.  With files on both sides:
//
//   reader threads   pull partition c's slices of every run into ring slot c mod R of the pinned INPUT ring -- as soon
//                    as the partition that used the slot before (c - R) has been consumed (its kernels are done)
//   engine thread    waits for partition c's reads, enqueues its H2D / kernels / D2H (into slot c mod R of the pinned
//                    OUTPUT ring, once partition c - R has left it), publishes what the D2H will deliver
//   writer threads   walk the partitions in order: wait for the D2H, push the slot's bytes through the write callback
//                    in pieces, hand the slot back
//
// so file reads, both PCIe directions and file writes all overlap, and the pinned memory is R slots however large the
// SSTables are.  Any callback error aborts the pump; the first error code is what every wait returns from then on.
//
// A partition's output is a list of pieces {destination, kind, file offset, bytes}: the compaction publishes two (its .data
// and .index), the streamed scan (dbeel_scan_stream) two per destination that received something.
#pragma once
#include <stdint.h>

#include <atomic>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "../../../include/dbeel_compact.h"

namespace dbeel {

class StreamPump {
  public:
    struct ReadTask {
        uint32_t part, run, kind;
        uint64_t off, len;
        uint8_t *dst;
    };
    struct OutPart { // where partition c's output sits in the pinned ring and where it goes in the files
        const uint8_t *data = nullptr;
        uint64_t data_len = 0, data_off = 0;
        const uint8_t *index = nullptr;
        uint64_t index_len = 0, index_off = 0;
    };
    struct OutPiece { // len bytes at src go to offset `off` of destination `dest`'s file of kind `kind` (DBEEL_STREAM_*)
        uint32_t dest, kind;
        uint64_t off;
        const uint8_t *src;
        uint64_t len;
    };
    static constexpr uint64_t kPiece = 8ull << 20; // bytes per callback call

    // wait_out(c): blocks until partition c's output has arrived in host memory (the engine: cudaEventSynchronize).
    // thread_init(): run once on every pump thread (the engine: cudaSetDevice).
    StreamPump(const dbeel_stream_io *io, uint32_t n_parts, uint32_t ring, int n_threads, std::function<void(uint32_t)> wait_out,
               std::function<void()> thread_init = nullptr)
        : StreamPump(io->read, io->write, nullptr, io->ctx, n_parts, ring, n_threads, std::move(wait_out), std::move(thread_init)) {}
    // The scan's callbacks: the same read, a write that names the destination.
    StreamPump(const dbeel_scan_io *io, uint32_t n_parts, uint32_t ring, int n_threads, std::function<void(uint32_t)> wait_out,
               std::function<void()> thread_init = nullptr)
        : StreamPump(io->read, nullptr, io->write, io->ctx, n_parts, ring, n_threads, std::move(wait_out), std::move(thread_init)) {}
    StreamPump(const StreamPump &) = delete;
    StreamPump &operator=(const StreamPump &) = delete;
    ~StreamPump() {
        abort(DBEEL_ERR_INVALID_ARG); // no-op for the error code when the pump finished cleanly
        join();
    }

    // Before start(), in partition order.  A slice longer than kPiece becomes several tasks.
    void add_read(uint32_t part, uint32_t run, uint32_t kind, uint64_t off, uint64_t len, uint8_t *dst) {
        for (uint64_t done = 0; done < len; done += kPiece) {
            const uint64_t n = len - done < kPiece ? len - done : kPiece;
            tasks_.push_back(ReadTask{part, run, kind, off + done, n, dst + done});
            r_left_[part]++;
        }
    }

    void start() {
        started_ = true;
        for (int i = 0; i < nt_; i++) threads_.emplace_back([this] { reader(); });
        for (int i = 0; i < nt_; i++) threads_.emplace_back([this] { writer(); });
    }

    int wait_reads(uint32_t part) {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return failed_ || r_left_[part] == 0; });
        return failed_ ? err_ : 0;
    }

    void release_input(uint32_t part) {
        std::lock_guard<std::mutex> lk(mu_);
        if (part + 1 > consumed_) consumed_ = part + 1;
        cv_.notify_all();
    }

    // The output ring slot of `part` is free once partition part - ring has been written out.
    int wait_out_slot(uint32_t part) {
        if (part < ring_) return 0;
        const uint32_t prev = part - ring_;
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return failed_ || (published_ > prev && w_left_[prev] == 0); });
        return failed_ ? err_ : 0;
    }

    void publish_out(uint32_t part, const OutPart &o) {
        publish_pieces(part, {OutPiece{0, DBEEL_STREAM_DATA, o.data_off, o.data, o.data_len},
                              OutPiece{0, DBEEL_STREAM_INDEX, o.index_off, o.index, o.index_len}});
    }

    // In partition order.  Pieces longer than kPiece go out in several callback calls.
    void publish_pieces(uint32_t part, std::vector<OutPiece> ps) {
        uint64_t calls = 0;
        for (const OutPiece &q : ps) calls += pieces(q.len);
        std::lock_guard<std::mutex> lk(mu_);
        outs_[part] = std::move(ps);
        w_total_[part] = calls;
        w_left_[part] = calls;
        published_ = part + 1;
        cv_.notify_all();
    }

    // Everything published has been written (or the pump failed).  Joins the threads.
    int finish() {
        {
            std::unique_lock<std::mutex> lk(mu_);
            cv_.wait(lk, [&] {
                if (failed_) return true;
                if (published_ < np_) return false;
                for (uint32_t c = 0; c < np_; c++)
                    if (w_left_[c]) return false;
                return true;
            });
            done_ = true;
            cv_.notify_all();
        }
        join();
        return failed_ ? err_ : 0;
    }

    void abort(int code) {
        std::lock_guard<std::mutex> lk(mu_);
        if (!failed_ && !done_) {
            failed_ = true;
            err_ = code;
        }
        cv_.notify_all();
    }

  private:
    using ReadFn = int (*)(void *, uint32_t, uint32_t, uint64_t, uint64_t, void *);
    using WriteFn = int (*)(void *, uint32_t, uint64_t, const void *, uint64_t);
    using WriteDestFn = int (*)(void *, uint32_t, uint32_t, uint64_t, const void *, uint64_t);

    StreamPump(ReadFn read, WriteFn write, WriteDestFn write_dest, void *ctx, uint32_t n_parts, uint32_t ring, int n_threads,
               std::function<void(uint32_t)> wait_out, std::function<void()> thread_init)
        : read_(read), write_(write), write_dest_(write_dest), ctx_(ctx), np_(n_parts), ring_(ring ? ring : 1), nt_(n_threads > 0 ? n_threads : 1),
          wait_out_(std::move(wait_out)), thread_init_(std::move(thread_init)), r_left_(n_parts, 0), w_total_(n_parts, 0), w_left_(n_parts, 0),
          w_next_(new std::atomic<uint64_t>[n_parts ? n_parts : 1]), outs_(n_parts) {
        for (uint32_t c = 0; c < n_parts; c++) w_next_[c].store(0);
    }

    static uint64_t pieces(uint64_t len) { return (len + kPiece - 1) / kPiece; }

    void join() {
        for (auto &t : threads_)
            if (t.joinable()) t.join();
        threads_.clear();
    }

    void fail_locked(int code) {
        if (!failed_) {
            failed_ = true;
            err_ = code ? code : DBEEL_ERR_INVALID_ARG;
        }
    }

    void reader() {
        if (thread_init_) thread_init_();
        while (true) {
            const size_t k = r_next_.fetch_add(1);
            if (k >= tasks_.size()) return;
            const ReadTask &t = tasks_[k];
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return failed_ || t.part < consumed_ + ring_; });
                if (failed_) return;
            }
            const int rc = read_(ctx_, t.run, t.kind, t.off, t.len, t.dst);
            std::lock_guard<std::mutex> lk(mu_);
            if (rc) fail_locked(rc);
            r_left_[t.part]--;
            cv_.notify_all();
            if (failed_) return;
        }
    }

    void writer() {
        if (thread_init_) thread_init_();
        for (uint32_t c = 0; c < np_; c++) {
            const std::vector<OutPiece> *ps;
            uint64_t total;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return failed_ || published_ > c; });
                if (failed_) return;
                ps = &outs_[c]; // neither changes once published
                total = w_total_[c];
            }
            if (total == 0) continue;
            if (wait_out_) wait_out_(c);
            size_t p = 0;      // the piece that holds call k (k only grows on this thread)
            uint64_t p0 = 0;   // calls of the pieces before it
            while (true) {
                const uint64_t k = w_next_[c].fetch_add(1);
                if (k >= total) break;
                while (k >= p0 + pieces((*ps)[p].len)) p0 += pieces((*ps)[p++].len);
                const OutPiece &o = (*ps)[p];
                const uint64_t off = (k - p0) * kPiece, n = o.len - off < kPiece ? o.len - off : kPiece;
                const int rc = write_dest_ ? write_dest_(ctx_, o.dest, o.kind, o.off + off, o.src + off, n)
                                           : write_(ctx_, o.kind, o.off + off, o.src + off, n);
                std::lock_guard<std::mutex> lk(mu_);
                if (rc) fail_locked(rc);
                w_left_[c]--;
                cv_.notify_all();
                if (failed_) return;
            }
        }
    }

    const ReadFn read_;
    const WriteFn write_;
    const WriteDestFn write_dest_;
    void *const ctx_;
    const uint32_t np_, ring_;
    const int nt_;
    std::function<void(uint32_t)> wait_out_;
    std::function<void()> thread_init_;
    std::vector<ReadTask> tasks_;
    std::atomic<size_t> r_next_{0};
    std::mutex mu_;
    std::condition_variable cv_;
    // all below under mu_
    std::vector<uint32_t> r_left_;
    std::vector<uint64_t> w_total_, w_left_; // callback calls of each partition's output: all / not yet done
    std::unique_ptr<std::atomic<uint64_t>[]> w_next_;
    std::vector<std::vector<OutPiece>> outs_;
    uint32_t consumed_ = 0;  // partitions [0, consumed_) have released their input slot
    uint32_t published_ = 0; // partitions [0, published_) have their output described
    bool failed_ = false, done_ = false, started_ = false;
    int err_ = 0;
    std::vector<std::thread> threads_;
};

} // namespace dbeel
