// bin/rsem-tbam2gbam: drop-in for the reference's tool of that name (tbam2gbam.cpp, BamConverter.h), which
// rsem-calculate-expression runs under --output-genome-bam (rsem-calculate-expression:649-653).
//
//   rsem-tbam2gbam reference_name unsorted_transcript_bam_input genome_bam_output [-p number_of_threads]
//
// Converts every alignment of a transcript BAM into genome coordinates with reference_name.ti (type 0) and
// reference_name.chrlist, and collapses the alignments of a read that land on the same genomic alignment into one
// record whose ZW is their sum.  Stdout, the header and the records are the reference's.
//
// The host reads the input (BGZF inflated on worker threads by AlnReader), frames it into units (a record, or a mate
// pair with mate 1 first) and groups (runs of mapped units of one read name; an unmapped unit is its own group) and
// checks what the reference checks while it reads (BamConverter.h:92-148).  Batches of whole groups go to the device
// (K10, csrc/gbam_kernels.cu), which converts, collapses and orders them.  Three things run at once: AlnReader's
// threads inflate the input ahead of the main thread, and a writer thread deflates the output of the previous batch
// (BamWriter).  The main thread frames a batch and then waits for its device call; framing does not overlap the device
// work, and the batch buffers are pageable host memory.
//
// -p N: threads for inflating and deflating.  Without -p (the driver never passes it) the count comes from
// RSEM_B200_IO_THREADS, else from the host's cores; the output does not depend on it.  RSEM_B200_GBAM_BATCH sets the
// batch size in bytes of input records (tests); a group larger than it makes a larger batch.  RSEM_B200_TIMING=1 prints
// the time of each phase to stderr.
//
// Differences: inputs the reference aborts on (a partial pair, a pair whose mates are on different transcripts, a
// mapped record with SEQ '*', an unmapped record that follows a record of the same name, a record the converter cannot
// place, a malformed .chrlist line) stop the run with a message and exit status 255; the reference asserts, crashes or
// exits -1 on them.  So does a read name with both single-end and paired-end records.
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <fstream>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "host.hpp"

using namespace host;

namespace {

double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// SamHeader::replaceSQ (SamHeader.cpp:30-46), including its substr(pos + 1, <index>) length; names -> output tid
std::string chrlist_sq(const std::string& path, std::map<std::string, int>& refmap) {
    std::ifstream fin(path.c_str());
    if (!fin.is_open()) die("Cannot open " + path + "! It may not exist.");
    std::string line, sq;
    int n = 0;
    while (getline(fin, line)) {
        const size_t pos = line.find_first_of('\t');
        if (pos == std::string::npos || pos == 0 || pos + 1 >= line.length() || line[pos + 1] == '\t')
            die("Malformed line in " + path + ": " + line);
        sq += "@SQ\tSN:" + line.substr(0, pos) + "\tLN:" + line.substr(pos + 1, line.find_first_of('\t', pos + 1)) + "\n";
        refmap[line.substr(0, pos)] = n++;
    }
    return sq;
}

std::string canonical_name(const BamRecord& b) {   // bam_get_canonical_name (sam_utils.h:54-61)
    const char* q = b.qname();
    return std::string(q, strcspn(q, " \t\n\r\f\v"));
}

struct Batch {
    std::vector<uint8_t> data;
    std::vector<uint64_t> rec_off;
    std::vector<uint32_t> unit_rec{0}, unit_group;
    std::vector<int32_t> unit_tr;
    uint32_t groups = 0;
    void clear() {
        data.clear();
        rec_off.clear();
        unit_rec.assign(1, 0);
        unit_group.clear();
        unit_tr.clear();
        groups = 0;
    }
    void add(const BamRecord& r) {
        rec_off.push_back(data.size());
        const uint32_t n = (uint32_t)r.data.size();
        const uint8_t b4[4] = {(uint8_t)n, (uint8_t)(n >> 8), (uint8_t)(n >> 16), (uint8_t)(n >> 24)};
        data.insert(data.end(), b4, b4 + 4);
        data.insert(data.end(), r.data.begin(), r.data.end());
    }
};

// deflates and writes the output of each batch on its own thread, one batch behind the reader
class Writer {
public:
    Writer(BamWriter& w) : w_(w), th_([this]() { run(); }) {}
    void push(std::vector<uint8_t>&& v) {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&]() { return q_.size() < 2; });
        q_.push_back(std::move(v));
        cv_.notify_all();
    }
    double finish() {
        { std::lock_guard<std::mutex> lk(mu_); done_ = true; }
        cv_.notify_all();
        th_.join();
        const double t0 = now();
        w_.close();
        return busy_ + (now() - t0);
    }
    std::vector<uint8_t> spare() {   // a consumed buffer to reuse, or an empty one
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<uint8_t> v;
        if (!spare_.empty()) { v.swap(spare_.back()); spare_.pop_back(); }
        return v;
    }

private:
    BamWriter& w_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<std::vector<uint8_t>> q_;
    std::vector<std::vector<uint8_t>> spare_;
    bool done_ = false;
    double busy_ = 0;
    std::thread th_;
    void run() {
        for (;;) {
            std::vector<uint8_t> v;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&]() { return !q_.empty() || done_; });
                if (q_.empty()) return;
                v = std::move(q_.front());
                q_.pop_front();
                cv_.notify_all();
            }
            const double t0 = now();
            w_.write_encoded(v.data(), v.size());
            busy_ += now() - t0;
            std::lock_guard<std::mutex> lk(mu_);
            spare_.push_back(std::move(v));
        }
    }
};

}  // namespace

int main(int argc, char* argv[]) {
    if (argc != 4 && argc != 6) {
        printf("Usage: rsem-tbam2gbam reference_name unsorted_transcript_bam_input genome_bam_output [-p number_of_threads]\n");
        exit(-1);
    }
    int threads = 0;
    if (argc == 6) {
        if (strcmp(argv[4], "-p") != 0) die("rsem-tbam2gbam: the fourth argument must be -p");
        threads = atoi(argv[5]);
    } else if (const char* e = getenv("RSEM_B200_IO_THREADS")) threads = atoi(e);
    else threads = (int)std::thread::hardware_concurrency();
    threads = std::max(1, threads);
    g_io_threads = threads;
    const std::string ref_name = argv[1];
    std::string command = argv[0];   // assemble_command (utils.h:159-164)
    for (int i = 1; i < argc; ++i) command += " " + std::string(argv[i]);

    const double t_start = now();
    std::vector<TranscriptInfo> tr;
    int ti_type = 0;
    load_transcripts(ref_name + ".ti", tr, &ti_type);
    const int M = (int)tr.size() - 1;
    printf("Start converting:\n");
    if (ti_type != 0) die("Genome information is not provided! RSEM cannot convert the transcript bam file!");

    AlnReader in(argv[2], "rsem-tbam2gbam");
    const std::vector<int> e2i = map_bam_targets(in.ref_names(), tr, ti_type);
    std::map<std::string, int> refmap;
    const std::string sq = chrlist_sq(ref_name + ".chrlist", refmap);
    const std::string header = rsem_bam_header_text(in.header_text(), "rsem-tbam2gbam", command, &sq, true);

    // transcript tables for the device, and the MAPQ thresholds
    std::vector<int32_t> out_tid(M + 1, -1), length(M + 1, 0);
    std::vector<uint8_t> minus(M + 1, 0);
    std::vector<int64_t> exon_off(M + 2, 0);
    std::vector<int32_t> exon_start, exon_end;
    size_t max_exons = 0;
    for (int t = 1; t <= M; ++t) {
        auto it = refmap.find(tr[t].seqname);
        if (it != refmap.end()) out_tid[t] = it->second;
        minus[t] = tr[t].strand == '-';
        length[t] = tr[t].length;
        for (auto& e : tr[t].exons) { exon_start.push_back(e.first); exon_end.push_back(e.second); }
        exon_off[t + 1] = (int64_t)exon_start.size();
        max_exons = std::max(max_exons, tr[t].exons.size());
    }
    const std::vector<float> mapq_prb = mapq_thresholds();
    rsem_b200_gbam_tables tables;
    memset(&tables, 0, sizeof tables);
    tables.M = M;
    tables.out_tid = out_tid.data();
    tables.minus = minus.data();
    tables.length = length.data();
    tables.exon_off = exon_off.data();
    tables.exon_start = exon_start.data();
    tables.exon_end = exon_end.data();
    tables.mapq_prb = mapq_prb.data();

    BamWriter bw(argv[3], header, threads);
    Writer writer(bw);
    rsem_b200_ctx* ctx = nullptr;
    const char* dev = getenv("RSEM_B200_DEVICE");
    size_t budget = 256u << 20;
    if (const char* e = getenv("RSEM_B200_GBAM_BATCH")) budget = std::max<size_t>(1, strtoull(e, nullptr, 10));

    Batch batch;
    double t_read = 0, t_device = 0, dev_ms = 0;
    uint64_t n_batches = 0;
    auto flush = [&]() {
        if (batch.unit_tr.empty()) return;
        const double t0 = now();
        if (!ctx) check_rc(rsem_b200_ctx_create(dev ? atoi(dev) : 0, &ctx), "ctx_create");
        // the converted records grow by their new CIGAR (at most 2 exons + 2 operations each) and one XS:A
        const size_t cap = batch.data.size() + batch.rec_off.size() * (8 * max_exons + 16);
        std::vector<uint8_t> out = writer.spare();
        out.resize(cap);
        rsem_b200_gbam_batch b;
        b.n_records = batch.rec_off.size();
        b.n_units = batch.unit_tr.size();
        b.n_bytes = batch.data.size();
        b.data = batch.data.data();
        b.rec_off = batch.rec_off.data();
        b.unit_rec = batch.unit_rec.data();
        b.unit_group = batch.unit_group.data();
        b.unit_tr = batch.unit_tr.data();
        uint64_t n_out = 0;
        rsem_b200_gbam_stats st;
        const int rc = rsem_b200_gbam_convert(ctx, &tables, &b, out.data(), out.size(), &n_out, &st);
        if (rc != 0 && st.bad_unit >= 0) {
            const uint8_t* r = batch.data.data() + batch.rec_off[batch.unit_rec[(size_t)st.bad_unit]] + 4;
            die(std::string("rsem-tbam2gbam: read ") + reinterpret_cast<const char*>(r + 32) + ": " + rsem_b200_last_error());
        }
        check_rc(rc, "gbam_convert");
        out.resize(n_out);
        dev_ms += st.device_ms;
        t_device += now() - t0;
        writer.push(std::move(out));
        batch.clear();
        ++n_batches;
    };

    BamRecord b, b2;
    std::string cqname, qname;
    bool have_cq = false, cq_paired = false;
    uint64_t cnt = 0;
    double t0 = now();
    while (in.next(b)) {
        ++cnt;
        const bool paired = b.paired();
        if (paired) {
            if (!in.next(b2) || !b2.paired()) die("rsem-tbam2gbam: read " + canonical_name(b) + " has a mate without the other");
            if (!b.read1()) std::swap(b, b2);
            if (!(b.read1() && b2.read2())) die("rsem-tbam2gbam: the mates of read " + canonical_name(b) + " are not read 1 and read 2");
            if (b.mapped() != b2.mapped())
                die("Detected partial alignments for read " + canonical_name(b) + ", which RSEM currently does not support!");
            ++cnt;
        }
        if (cnt % 1000000 == 0) { printf("."); fflush(stdout); }
        qname = canonical_name(b);
        const bool same = have_cq && cqname == qname;
        if (same && paired != cq_paired) die("rsem-tbam2gbam: read " + qname + " has both single-end and paired-end records");
        int t = 0;
        if (b.mapped()) {
            if (paired && b.tid() != b2.tid()) die(qname + "'s two mates are aligned to two different transcripts!");
            if (b.tid() < 0 || b.tid() >= (int32_t)e2i.size()) die("rsem-tbam2gbam: read " + qname + " is mapped to no transcript");
            if (b.l_seq() <= 0 || (paired && b2.l_seq() <= 0)) die("One alignment line has SEQ field as *. RSEM does not support this currently!");
            t = e2i[(size_t)b.tid()];
        } else if (same) {
            die("rsem-tbam2gbam: an unmapped record of read " + qname + " follows another record of that read");
        }
        // a new name starts a group; so does a mapped unit after an unmapped one of the same name, because the reference
        // has cleared its CollapseMap there (BamConverter.h:136-146).  Batches are cut at group starts only.
        if (!same || batch.unit_tr.back() == 0) {
            if (batch.data.size() >= budget) {
                t_read += now() - t0;
                flush();
                t0 = now();
            }
            ++batch.groups;
        }
        batch.unit_group.push_back(batch.groups - 1);
        batch.unit_tr.push_back(t);
        batch.add(b);
        if (paired) batch.add(b2);
        batch.unit_rec.push_back((uint32_t)batch.rec_off.size());
        cqname = qname;
        have_cq = true;
        cq_paired = paired;
    }
    t_read += now() - t0;
    flush();
    const double t_write = writer.finish();
    if (ctx) rsem_b200_ctx_destroy(ctx);
    if (cnt >= 1000000) printf("\n");
    printf("Genome bam file is generated!\n");
    if (getenv("RSEM_B200_TIMING"))
        fprintf(stderr,
                "rsem-tbam2gbam timing: total %.3f s; read+inflate+frame %.3f s, device calls %.3f s (device %.3f s), "
                "deflate+write %.3f s (on its own thread); %llu records, %llu batches, %d threads\n",
                now() - t_start, t_read, t_device, dev_ms / 1e3, t_write, (unsigned long long)cnt,
                (unsigned long long)n_batches, threads);
    return 0;
}
