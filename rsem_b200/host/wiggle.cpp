// Shared code of bin/rsem-bam2wig and bin/rsem-bam2readdepth: build_wiggles (wiggle.cpp:16-83) with the per-base sums
// on the device (K11, csrc/wiggle_kernels.cu) and the two writers (wiggle.cpp:85-130) on host threads.
//
// The main thread reads the input (BGZF inflated on AlnReader's threads), keeps the mapped records and frames them into
// batches of whole records: runs of one target, the last of which may continue into the next batch (its depth stays on
// the device).  After each device call it formats the targets the call finished, in position chunks on
// RSEM_B200_IO_THREADS threads (default: the host's cores), and hands the text to a writer thread, which writes one
// chunk behind.  The output does not depend on the thread count or the batch size (RSEM_B200_WIG_BATCH, bytes of
// records; tests force many batches with it).  An input without mapped records needs no device.
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "host.hpp"

namespace host {

namespace {

double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct Piece {            // positions [a, b) of one target
    size_t t;
    uint64_t a, b;
};

void format_piece(const WigTarget& T, const Piece& p, bool wig, std::string& s) {
    char buf[512];   // %.2f of the largest double is 313 characters with its newline
    if (wig) {   // UCSCWiggleTrackWriter::process: runs of depth >= 0.0095, each after its fixedStep line
        const double* d = T.depth;
        if (!d) return;
        for (uint64_t i = p.a; i < p.b; ++i) {
            if (!(d[i] >= 0.0095)) continue;
            if (i == 0 || !(d[i - 1] >= 0.0095)) {
                s += "fixedStep chrom=";
                s += T.name;
                snprintf(buf, sizeof buf, " start=%d step=1\n", (int)i + 1);
                s += buf;
            }
            const int n = snprintf(buf, sizeof buf, "%.2f\n", d[i]);
            s.append(buf, (size_t)n);
        }
        return;
    }
    // ReadDepthWriter::process: name, length, then every value as ostream << double prints it (%.6g), or NA
    if (p.a == 0) {
        s += T.name;
        snprintf(buf, sizeof buf, "\t%llu\t", (unsigned long long)T.length);
        s += buf;
        if (!T.depth || T.length == 0) {
            s += "NA\n";
            return;
        }
    }
    const double* d = T.depth;
    for (uint64_t i = p.a; i < p.b; ++i) {
        if (i > 0) s += ' ';
        if (__builtin_expect(d[i] == 0.0 && !std::signbit(d[i]), 1)) {
            s += '0';
            continue;
        }
        const int n = snprintf(buf, sizeof buf, "%.*g", 6, d[i]);
        s.append(buf, (size_t)n);
    }
    if (p.b == T.length) s += '\n';
}

// hands each call's formatted chunks to a thread that writes them in order, one call behind the main thread
class Writer {
public:
    explicit Writer(FILE* f) : f_(f), th_([this]() { run(); }) {}
    void push(std::vector<std::string>&& v) {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&]() { return q_.size() < 2; });
        q_.push_back(std::move(v));
        cv_.notify_all();
    }
    double finish() {   // writes what is queued; -> seconds spent writing
        {
            std::lock_guard<std::mutex> lk(mu_);
            if (done_) return busy_;
            done_ = true;
        }
        cv_.notify_all();
        th_.join();
        return busy_;
    }
    bool failed() const { return failed_; }

private:
    FILE* f_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<std::vector<std::string>> q_;
    bool done_ = false, failed_ = false;
    double busy_ = 0;
    std::thread th_;
    void run() {
        for (;;) {
            std::vector<std::string> v;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&]() { return !q_.empty() || done_; });
                if (q_.empty()) return;
                v = std::move(q_.front());
                q_.pop_front();
                cv_.notify_all();
            }
            const double t0 = now();
            for (const std::string& s : v)
                if (!s.empty() && fwrite(s.data(), 1, s.size(), f_) != s.size()) failed_ = true;
            busy_ += now() - t0;
        }
    }
};

}  // namespace

void format_wiggles(const std::vector<WigTarget>& targets, bool wig, size_t chunk_positions, int threads,
                    std::vector<std::string>& chunks) {
    chunk_positions = std::max<size_t>(chunk_positions, 1);
    // pieces of at most chunk_positions positions, grouped into chunks of about that many (a target without values
    // weighs one position)
    std::vector<std::vector<Piece>> plan(1);
    size_t fill = 0;
    for (size_t t = 0; t < targets.size(); ++t) {
        const WigTarget& T = targets[t];
        const uint64_t len = T.depth ? T.length : 0;
        uint64_t a = 0;
        do {
            const uint64_t b = std::min<uint64_t>(len, a + (chunk_positions - fill));
            plan.back().push_back(Piece{t, a, b});
            fill += std::max<uint64_t>(b - a, 1);
            if (fill >= chunk_positions) {
                plan.emplace_back();
                fill = 0;
            }
            a = b;
        } while (a < len);
    }
    if (plan.back().empty()) plan.pop_back();
    chunks.assign(plan.size(), std::string());
    parallel_ranges(plan.size(), std::max(1, std::min<int>(threads, (int)plan.size())), [&](size_t lo, size_t hi, int) {
        for (size_t c = lo; c < hi; ++c)
            for (const Piece& p : plan[c]) format_piece(targets[p.t], p, wig, chunks[c]);
    });
}

void run_wiggles(const char* tool, const std::string& in_path, bool wig, bool no_fractional_weight, FILE* out) {
    const double t_start = now();
    {   // sam_open's failure (wiggle.cpp:49): htslib 1.3's message, then the reference's
        FILE* probe = fopen(in_path.c_str(), "rb");
        if (!probe) {
            fprintf(stderr, "[E::hts_open_format] fail to open file '%s'\n", in_path.c_str());
            die("Cannot open " + in_path + "!");
        }
        fclose(probe);
    }
    AlnReader in(in_path, tool, true);
    const std::vector<std::string>& names = in.ref_names();
    const std::vector<uint32_t>& lens = in.ref_lens();
    const size_t n_targets = names.size();
    std::vector<char> used(n_targets, 0);
    const int threads = g_io_threads;
    size_t budget = 64u << 20;
    if (const char* e = getenv("RSEM_B200_WIG_BATCH")) budget = std::max<size_t>(1, strtoull(e, nullptr, 10));
    const uint64_t pos_budget = 1ull << 28;   // positions of the runs of one batch (device depth: 8 bytes each)
    const size_t chunk_positions = 1u << 16;
    Writer writer(out);
    rsem_b200_ctx* ctx = nullptr;
    const char* dev = getenv("RSEM_B200_DEVICE");

    // the batch being framed
    std::vector<uint8_t> data;
    std::vector<uint64_t> rec_off;
    std::vector<uint32_t> rec_run, run_len;
    std::vector<int32_t> run_tid;
    uint64_t run_positions = 0;
    uint64_t cnt = 0, batch_cnt0 = 0;   // mapped records read; and before the batch's first record
    int cur_tid = -1;                   // the open target: the last run of the batch, or the resident run
    bool resident = false;              // the device holds the open target's run from an earlier call
    int32_t resident_tid = -1;
    std::vector<double> depth;
    double t_read = 0, t_device = 0, dev_ms = 0, t_format = 0;
    uint64_t n_calls = 0;

    auto stop = [&](const std::string& msg) {
        writer.finish();
        fflush(out);
        die(msg);
    };
    auto progress = [&](uint64_t upto) {   // the reference's progress lines for the counts in (batch_cnt0, upto]
        for (uint64_t c = (batch_cnt0 / 1000000 + 1) * 1000000; c <= upto; c += 1000000) printf("%llu\n", (unsigned long long)c);
        fflush(stdout);
    };
    // the targets one call finished, formatted and queued for the writer
    auto emit = [&](const std::vector<int32_t>& tids, const double* d) {
        const double t0 = now();
        std::vector<WigTarget> ts(tids.size());
        uint64_t at = 0;
        for (size_t k = 0; k < tids.size(); ++k) {
            ts[k].name = names[(size_t)tids[k]];
            ts[k].length = lens[(size_t)tids[k]];
            ts[k].depth = ts[k].length ? d + at : nullptr;
            at += ts[k].length;
        }
        std::vector<std::string> chunks;
        format_wiggles(ts, wig, chunk_positions, threads, chunks);
        t_format += now() - t0;
        writer.push(std::move(chunks));
    };
    // one device call on the framed batch; final: the last run is finished too (and a resident run with no batch)
    bool batch_continues = false;       // run 0 of the batch is the resident run
    auto call = [&](bool final) {
        const uint32_t R = (uint32_t)run_len.size();
        if (R == 0 && !(final && resident)) return;
        const double t0 = now();
        if (!ctx) check_rc(rsem_b200_ctx_create(dev ? atoi(dev) : 0, &ctx), "ctx_create");
        std::vector<int32_t> done;
        uint64_t cap = 0;
        if (resident && !batch_continues) {
            done.push_back(resident_tid);
            cap += lens[(size_t)resident_tid];
        }
        for (uint32_t i = 0; i < R; ++i) {
            if (final || i + 1 < R) done.push_back(run_tid[i]);
            cap += run_len[i];
        }
        depth.resize(cap);
        rsem_b200_wig_batch b;
        memset(&b, 0, sizeof b);
        b.n_records = rec_off.size();
        b.n_bytes = data.size();
        b.data = data.data();
        b.rec_off = rec_off.data();
        b.rec_run = rec_run.data();
        b.run_len = run_len.data();
        b.n_runs = R;
        b.continues = batch_continues ? 1 : 0;
        b.keep_last = final ? 0 : 1;
        b.no_fractional_weight = no_fractional_weight ? 1 : 0;
        uint64_t got = 0;
        rsem_b200_wig_stats st{0.0, 0, 0, -1, 0, 0};
        const int rc = rsem_b200_wig_depth(ctx, &b, depth.data(), depth.size(), &got, &st);
        if (rc != 0 && st.bad_record >= 0) {
            progress(batch_cnt0 + (uint64_t)st.bad_record);
            const uint8_t* r = data.data() + rec_off[(size_t)st.bad_record] + 4;
            stop(std::string(tool) + ": read " + reinterpret_cast<const char*>(r + 32) + ": " + rsem_b200_last_error());
        }
        if (rc != 0) {
            writer.finish();
            check_rc(rc, "wig_depth");
        }
        dev_ms += st.device_ms;
        ++n_calls;
        t_device += now() - t0;
        progress(cnt);
        emit(done, depth.data());
        resident = !final && R > 0;
        resident_tid = resident ? run_tid.back() : -1;
        data.clear();
        rec_off.clear();
        rec_run.clear();
        run_len.clear();
        run_tid.clear();
        run_positions = 0;
        batch_cnt0 = cnt;
        batch_continues = false;
    };

    BamRecord rec;
    double t0 = now();
    auto cut = [&](bool final) {
        t_read += now() - t0;
        call(final);
        t0 = now();
    };
    while (in.next(rec)) {
        if (!rec.mapped()) continue;   // bam_is_unmapped (sam_utils.h:50)
        const int32_t tid = rec.tid();
        const int32_t pos = rec.pos();
        if (tid < 0 || (size_t)tid >= n_targets || pos < 0) {
            cut(false);
            stop(std::string(tool) + ": read " + rec.qname() +
                 (pos < 0 && tid >= 0 && (size_t)tid < n_targets
                      ? ": a mapped record with a negative position (reference: writes before its depth vector)"
                      : ": a mapped record whose target is not in the header (reference: reads past its target table)"));
        }
        if (tid != cur_tid) {   // a new target opens (wiggle.cpp:61-67)
            if (!rec_off.empty() && (data.size() >= budget || run_positions + lens[(size_t)tid] > pos_budget)) cut(false);
            if (cur_tid >= 0) used[(size_t)cur_tid] = 1;
            cur_tid = tid;
            run_len.push_back(lens[(size_t)tid]);
            run_tid.push_back(tid);
            run_positions += lens[(size_t)tid];
        } else if (data.size() >= budget) {   // the open target continues in the next batch
            cut(false);
            batch_continues = true;
            run_len.push_back(lens[(size_t)tid]);
            run_tid.push_back(tid);
            run_positions += lens[(size_t)tid];
        }
        rec_off.push_back(data.size());
        const uint32_t n = (uint32_t)rec.data.size();
        const uint8_t b4[4] = {(uint8_t)n, (uint8_t)(n >> 8), (uint8_t)(n >> 16), (uint8_t)(n >> 24)};
        data.insert(data.end(), b4, b4 + 4);
        data.insert(data.end(), rec.data.begin(), rec.data.end());
        rec_run.push_back((uint32_t)run_len.size() - 1);
        ++cnt;
    }
    cut(true);
    if (cur_tid >= 0) used[(size_t)cur_tid] = 1;
    {   // targets never opened, in header order, with an empty read_depth (wiggle.cpp:71-77)
        std::vector<int32_t> rest;
        for (size_t i = 0; i < n_targets; ++i)
            if (!used[i]) rest.push_back((int32_t)i);
        if (!rest.empty()) {
            const double t1 = now();
            std::vector<WigTarget> ts(rest.size());
            for (size_t k = 0; k < rest.size(); ++k) {
                ts[k].name = names[(size_t)rest[k]];
                ts[k].length = lens[(size_t)rest[k]];
            }
            std::vector<std::string> chunks;
            format_wiggles(ts, wig, chunk_positions, threads, chunks);
            t_format += now() - t1;
            writer.push(std::move(chunks));
        }
    }
    const double t_write = writer.finish();
    if (ctx) rsem_b200_ctx_destroy(ctx);
    if (writer.failed()) die(std::string(tool) + ": cannot write the output");
    if (getenv("RSEM_B200_TIMING"))
        fprintf(stderr,
                "%s timing: total %.3f s; read+frame %.3f s, device calls %.3f s (device %.3f s), format %.3f s, "
                "write %.3f s (on its own thread); %llu mapped records, %llu device calls, %d threads\n",
                tool, now() - t_start, t_read, t_device, dev_ms / 1e3, t_format, t_write, (unsigned long long)cnt,
                (unsigned long long)n_calls, threads);
}

}  // namespace host
