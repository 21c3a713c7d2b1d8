// rsem-parse-alignments, H100 edition: the caller-side hand-off of the hot path (SURVEY.md 8(f).2).
//
//   rsem-parse-alignments refName imdName statName alignF read_type [-t fai_file] [-tag tagName] [-q]
//
// Same argv, same output files as the reference executable (/root/reference/parseIt.cpp:172-229, SamParser.h):
// imdName.dat (hits per alignable read), imdName_{un,alignable,max}[_1,_2].{fa,fq} (the reads by category),
// statName.cnt (alignment statistics) and imdName.omit (transcripts the alignment file does not declare) are
// byte-identical to the reference's, so the unmodified rsem-calculate-expression, rsem-build-read-index and the
// reference's own rsem-run-em keep working on them.  In the same pass the decoded content is kept in the layout
// bin/rsem-run-em uploads to the GPU (CSR + SoA hit fields, base / quality codes) and written as the binary side-car
// imdName.b200 (host/sidecar.cpp): rsem-run-em then skips its text parse of .dat and of the read files.
//
// SAM (plain / gzip) and BAM are read with this repository's own reader (host/bam.cpp); CRAM and `-t fai_file`
// (only meaningful for CRAM / header-less SAM in htslib) are not supported.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <deque>
#include <map>
#include <mutex>
#include <thread>

#include "host.hpp"

using namespace host;

namespace {

// Text output: every file appends to a 4 MB buffer; full buffers go to ONE background writer thread (FIFO, so the order per
// file is kept), which keeps the write syscalls off the parsing thread.  Files of categories that stayed empty are removed at
// the end (parseIt.cpp:158-170).
class Writer {
public:
    Writer() : th_([this]() { run(); }) {}
    ~Writer() { finish(); }
    void submit(FILE* f, const std::string* path, std::string&& data) {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&]() { return q_.size() < 16; });
        q_.push_back(Job{f, path, std::move(data)});
        cv_.notify_all();
    }
    std::string spare() {   // an emptied buffer with its capacity, if one is available
        std::lock_guard<std::mutex> lk(mu_);
        if (spare_.empty()) return std::string();
        std::string s = std::move(spare_.back());
        spare_.pop_back();
        return s;
    }
    void drain() {   // everything submitted so far is on its way to the kernel
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&]() { return q_.empty() && !busy_; });
    }
    void finish() {
        if (!th_.joinable()) return;
        { std::lock_guard<std::mutex> lk(mu_); stop_ = true; }
        cv_.notify_all();
        th_.join();
    }

private:
    struct Job { FILE* f; const std::string* path; std::string data; };
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<Job> q_;
    std::vector<std::string> spare_;
    bool stop_ = false, busy_ = false;
    std::thread th_;
    void run() {
        for (;;) {
            Job j;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&]() { return !q_.empty() || stop_; });
                if (q_.empty()) return;
                j = std::move(q_.front());
                q_.pop_front();
                busy_ = true;
                cv_.notify_all();
            }
            if (fwrite(j.data.data(), 1, j.data.size(), j.f) != j.data.size()) die("Cannot write " + *j.path + " (disk full?)!");
            j.data.clear();
            std::lock_guard<std::mutex> lk(mu_);
            if (spare_.size() < 8) spare_.push_back(std::move(j.data));
            busy_ = false;
            cv_.notify_all();
        }
    }
};

struct OutFile {
    std::string path;
    FILE* f = nullptr;
    std::string buf;
    Writer* w = nullptr;
    void open(const std::string& p, Writer* writer) {
        path = p;
        w = writer;
        f = fopen(p.c_str(), "w");
        if (!f) die("Cannot open " + p + " for writing!");
        buf.reserve(1 << 22);
    }
    void flush() {
        if (buf.empty()) return;
        w->submit(f, &path, std::move(buf));
        buf = w->spare();
        buf.clear();
        if (buf.capacity() < (1u << 22)) buf.reserve(1 << 22);
    }
    void put(const char* p, size_t n) {
        buf.append(p, n);
        if (buf.size() >= (1u << 22) - 4096) flush();
    }
    void put(const std::string& s) { put(s.data(), s.size()); }
    void put(char c) { buf.push_back(c); }
    void close() {   // after Writer::drain()
        if (fclose(f) != 0) die("Cannot write " + path + " (disk full?)!");
        f = nullptr;
    }
};

struct Mate {
    std::string name, seq, qual;
};
struct Read {   // SingleRead(Q) / PairedEndRead(Q) as parseIt keeps them between alignment lines
    std::string name;   // Read::name: the (first mate's) canonical name
    Mate mate[2];
};
struct Hit { int32_t sid, pos, insertL; };

const char* kWhitespace = " \t\n\r\f\v";

// decimal text of v at p, returns the new end (the .dat body is ~10 such numbers per alignment)
inline char* put_int(char* p, long long v) {
    if (v < 0) { *p++ = '-'; v = -v; }
    char tmp[24];
    int n = 0;
    do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) *p++ = tmp[--n];
    return p;
}

// length of the canonical read name: the first whitespace-delimited word of QNAME (sam_utils.h:58-65)
inline size_t canonical_len(const char* raw) { return strcspn(raw, kWhitespace); }

// sam_utils.h:58-65: only the first whitespace-delimited word of QNAME
std::string canonical_name(const BamRecord& b) {
    const char* raw = b.qname();
    return std::string(raw, canonical_len(raw));
}

// sam_utils.h:78-117: the read as it was sequenced (reverse-complemented back for reverse-strand alignments)
void read_seq(const BamRecord& b, std::string& out) {
    static const char fwd[17] = "\0AC\0G\0\0\0T\0\0\0\0\0\0N", rvs[17] = "\0TG\0C\0\0\0A\0\0\0\0\0\0N";
    const int n = b.l_seq();
    out.resize((size_t)n);
    const bool rev = b.reverse();
    const char* lut = rev ? rvs : fwd;
    char bad = 1;
    for (int i = 0; i < n; ++i) {
        const char c = lut[b.base4(rev ? n - 1 - i : i)];
        bad &= c != 0;
        out[(size_t)i] = c;
    }
    if (!bad) die("Read " + canonical_name(b) + " contains a base other than A, C, G, T and N (reference: assert(false) in bam_get_read_seq)!");
}

// sam_utils.h:119-139
void read_qual(const BamRecord& b, std::string& out) {
    const int n = b.l_seq();
    const uint8_t* q = b.qual();
    out.resize((size_t)n);
    if (b.reverse()) for (int i = 0; i < n; ++i) out[(size_t)i] = (char)(q[n - 1 - i] + 33);
    else for (int i = 0; i < n; ++i) out[(size_t)i] = (char)(q[i] + 33);
}

// sam_utils.h:68-75: one M / = / X operation covering the whole read
bool cigar_ok(const BamRecord& b) {
    if (b.n_cigar() != 1) return false;
    const uint32_t c = b.cigar(0), op = c & 15;
    return (op == 0 || op == 7 || op == 8) && (int32_t)(c >> 4) == b.l_seq();
}

struct Parser {
    int read_type = 0;
    bool hasq = false, paired = false;
    std::string rt_tag;   // -tag: the aligner's "too many alignments" tag (SamParser.h:58-81)
    AlnReader* in = nullptr;
    std::vector<int> e2i;   // external (header order, 0-based) -> internal transcript id
    BamRecord b, b2;
    int n_warns = 0;

    int tag_type(const BamRecord& r) const {   // 0 no tag / value <= 0, 2 otherwise
        if (rt_tag.empty()) return 0;
        long long v = 0;
        return (r.aux_int(rt_tag.c_str(), v) && v > 0) ? 2 : 0;
    }
    int internal_sid(const BamRecord& r) const {
        const int32_t t = r.tid();
        if (t < 0 || t >= (int32_t)e2i.size()) die("Read " + canonical_name(r) + " aligns to a reference sequence the header does not declare!");
        return e2i[(size_t)t];
    }

    // SamParser::parseNext: -1 end of input, 0/1/2 a new read of that category, 5 another alignment of the same read
    int next(Read& read, Hit& hit) {
        if (!paired) {
            if (!in->next(b)) return -1;
            const char* raw = b.qname();
            const size_t nlen = canonical_len(raw);
            if (b.paired()) die("Read " + std::string(raw, nlen) + ": Find a paired end read in the file!");
            const int type = b.mapped() ? 1 : tag_type(b);
            int val;
            if (type != 1 || read.name.size() != nlen || memcmp(read.name.data(), raw, nlen) != 0) {
                val = type;
                const std::string name(raw, nlen);
                read.name = name;
                read.mate[0].name = name;
                read_seq(b, read.mate[0].seq);
                if (hasq) read_qual(b, read.mate[0].qual);
            } else {
                if ((int)read.mate[0].seq.size() != b.l_seq()) die("Read " + std::string(raw, nlen) + " has alignments with inconsistent read lengths!");
                val = 5;
            }
            if (type == 1) {
                if (!cigar_ok(b)) die("Read " + std::string(raw, nlen) + ": RSEM currently does not support gapped alignments, sorry!\n");
                const int sid = internal_sid(b);
                if (b.reverse()) hit = Hit{-sid, (int32_t)in->ref_lens()[(size_t)b.tid()] - b.pos() - b.l_seq(), 0};
                else hit = Hit{sid, b.pos(), 0};
            }
            return val;
        }
        if (!in->next(b) || !in->next(b2)) return -1;
        if (!b.read1()) b.data.swap(b2.data);
        const char* raw = b.qname();
        const size_t nlen = canonical_len(raw);
        const char* raw2 = b2.qname();
        const size_t nlen2 = canonical_len(raw2);
        auto name_of = [&]() { return std::string(raw, nlen); };
        if (!(b.paired() && b2.paired()))
            die("Read " + name_of() + ": One of the mate is not paired-end! (RSEM assumes the two mates of a paired-end read should be adjacent)");
        if (!(b.read1() && b2.read2()))
            die("Read " + name_of() + ": The adjacent two lines do not represent the two mates of a paired-end read! (RSEM assumes the two mates of a paired-end read should be adjacent)");
        if (b.mapped() != b2.mapped()) die("Read " + name_of() + ": RSEM currently does not support partial alignments!");
        if ((nlen != nlen2 || memcmp(raw, raw2, nlen) != 0) && ++n_warns <= 50)   // MAX_WARNS, utils.h
            fprintf(stderr, "Warning: Detected a read pair whose two mates have different names--%s and %s!\n", name_of().c_str(),
                    std::string(raw2, nlen2).c_str());
        int type;
        if (b.mapped() && b2.mapped()) type = 1;
        else type = (tag_type(b) == 2 || tag_type(b2) == 2) ? 2 : 0;
        int val;
        if (type != 1 || read.name.size() != nlen || memcmp(read.name.data(), raw, nlen) != 0) {
            val = type;
            const std::string name = name_of();
            read.name = name;
            read.mate[0].name = name;
            read.mate[1].name.assign(raw2, nlen2);
            read_seq(b, read.mate[0].seq);
            read_seq(b2, read.mate[1].seq);
            if (hasq) { read_qual(b, read.mate[0].qual); read_qual(b2, read.mate[1].qual); }
        } else {
            if (!((int)read.mate[0].seq.size() == b.l_seq() && (int)read.mate[1].seq.size() == b2.l_seq()))
                die("Paired-end read " + name_of() + " has alignments with inconsistent mate lengths!");
            val = 5;
        }
        if (type == 1) {
            if (!(cigar_ok(b) && cigar_ok(b2))) die("Read " + name_of() + ": RSEM currently does not support gapped alignments, sorry!");
            if (b.tid() != b2.tid()) die("Read " + name_of() + ": The two mates do not align to a same transcript! RSEM does not support discordant alignments.");
            const int sid = internal_sid(b);
            if (b.reverse())
                hit = Hit{-sid, (int32_t)in->ref_lens()[(size_t)b.tid()] - b.pos() - b.l_seq(), b.pos() + b.l_seq() - b2.pos()};
            else
                hit = Hit{sid, b.pos(), b2.pos() + b2.l_seq() - b.pos()};
        }
        return val;
    }
};

int8_t g_base_code[256];

void append_read(ReadStore& rs, std::vector<ShortRead>& shorts, const Read& r, int n_mates, bool hasq) {
    bool is_short = false;
    for (int m = 0; m < n_mates; ++m) {
        const Mate& mt = r.mate[m];
        if (rs.off[m].empty()) rs.off[m].push_back(0);
        const size_t n = mt.seq.size(), at = rs.base[m].size();
        rs.base[m].resize(at + n);
        uint8_t* bd = rs.base[m].data() + at;
        for (size_t k = 0; k < n; ++k) bd[k] = (uint8_t)g_base_code[(unsigned char)mt.seq[k]];
        if (hasq) {
            rs.qual[m].resize(at + n);
            uint8_t* qd = rs.qual[m].data() + at;
            for (size_t k = 0; k < n; ++k) qd[k] = (uint8_t)((unsigned char)mt.qual[k] - 33);
        }
        rs.off[m].push_back(rs.off[m].back() + mt.seq.size());
        is_short = is_short || (int)mt.seq.size() < kSidecarShortLen;
    }
    if (is_short) shorts.push_back(ShortRead{rs.n, r.mate[0].name});   // the text path reports the first file's header line
    ++rs.n;
}

}  // namespace

int main(int argc, char* argv[]) {
    if (argc < 6) {
        printf("Usage : rsem-parse-alignments refName imdName statName alignF read_type [-t fai_file] [-tag tagName] [-q]\n");
        exit(-1);
    }
    const std::string refName = argv[1], imdName = argv[2], statName = argv[3], alignF = argv[4];
    const int read_type = atoi(argv[5]);
    Parser ps;
    for (int i = 6; i < argc; ++i) {
        if (!strcmp(argv[i], "-t") && i + 1 < argc)
            fprintf(stderr, "Warning: rsem-parse-alignments (H100): -t %s is ignored (a FASTA index is only needed for CRAM, which is not supported).\n", argv[i + 1]);
        if (!strcmp(argv[i], "-tag") && i + 1 < argc) ps.rt_tag = argv[i + 1];
        if (!strcmp(argv[i], "-q")) g_verbose = false;
    }
    if (read_type < 0 || read_type > 3) die("Unknown Read Type!");
    {   // the reference has no -p here; host threads inflate the BGZF blocks of the input (RSEM_B200_IO_THREADS, default <= 8)
        const char* e = getenv("RSEM_B200_IO_THREADS");
        g_io_threads = e ? std::max(1, atoi(e)) : (int)std::max(1u, std::min(8u, std::thread::hardware_concurrency()));
    }
    if (!ps.rt_tag.empty() && ps.rt_tag.size() != 2) die("-tag expects a two-character SAM tag!");
    ps.read_type = read_type;
    ps.hasq = read_type & 1;
    ps.paired = read_type >= 2;
    const int n_os = ps.paired ? 2 : 1;
    memset(g_base_code, 4, sizeof g_base_code);
    g_base_code[(unsigned char)'A'] = 0; g_base_code[(unsigned char)'C'] = 1; g_base_code[(unsigned char)'G'] = 2; g_base_code[(unsigned char)'T'] = 3;

    std::vector<int> starts;
    load_groups(refName + ".grp", starts);
    std::vector<int> gid((size_t)starts.back(), 0);   // GroupInfo.h:49-56
    for (size_t g = 0; g + 1 < starts.size(); ++g) for (int j = starts[g]; j < starts[g + 1]; ++j) gid[(size_t)j] = (int)g;
    std::vector<TranscriptInfo> tr;
    int ti_type = 0;
    load_transcripts(refName + ".ti", tr, &ti_type);
    const int M = (int)tr.size() - 1;

    // SamParser constructor + Transcripts::buildMappings (Transcripts.h:105-143): header order -> internal ids, imd.omit
    AlnReader in(alignF);
    ps.in = &in;
    {
        const std::vector<std::string>& names = in.ref_names();
        if (names.empty()) die("The SAM/BAM file declares less than one reference sequence!");
        if ((int)names.size() > M) die("The SAM/BAM file declares more reference sequences (" + std::to_string(names.size()) + ") than RSEM knows (" + std::to_string(M) + ")!");
        if ((int)names.size() < M)
            fprintf(stderr, "Warning: The SAM/BAM file declares less reference sequences (%d) than RSEM knows (%d)! Please make sure that you aligned your reads against transcript sequences instead of genome.\n", (int)names.size(), M);
        std::map<std::string, int> dict;
        for (int i = 1; i <= M; ++i) {
            const std::string& tid = ti_type == 2 ? tr[i].seqname : tr[i].transcript_id;
            if (!dict.emplace(tid, i).second) die("RSEM's indices might be corrupted, " + tid + " appears more than once!");
        }
        std::vector<bool> appeared((size_t)M + 1, false);
        ps.e2i.assign(names.size(), 0);
        for (size_t i = 0; i < names.size(); ++i) {
            auto it = dict.find(names[i]);
            if (it == dict.end()) die("RSEM can not recognize reference sequence name " + names[i] + "!");
            if (it->second < 0) die("Reference sequence name " + names[i] + " appears more than once in the SAM/BAM file!");
            ps.e2i[i] = it->second;
            appeared[(size_t)it->second] = true;
            it->second = -1;
        }
        FILE* fo = fopen((imdName + ".omit").c_str(), "w");
        if (!fo) die("Cannot open " + imdName + ".omit for writing!");
        for (int i = 1; i <= M; ++i) if (!appeared[(size_t)i]) fprintf(fo, "%d\n", i);
        fclose(fo);
    }

    Writer writer;
    OutFile cat[3][2];
    for (int t = 0; t < 3; ++t) {
        std::vector<std::string> files;
        read_type_files(imdName, t, read_type, files);
        for (int m = 0; m < n_os; ++m) cat[t][m].open(files[(size_t)m], &writer);
    }
    OutFile dat;
    dat.open(imdName + ".dat", &writer);
    dat.put(std::string(99, ' '));   // room for the header, filled in at the end (parseIt.cpp:197-199, 208-209)
    dat.put('\n');

    Sidecar sc;
    sc.read_type = read_type;
    for (int t = 0; t < 3; ++t) { sc.reads[t].n_mates = n_os; sc.reads[t].has_qual = ps.hasq; for (int m = 0; m < n_os; ++m) sc.reads[t].off[m].assign(1, 0); }
    sc.hits.row_ptr.assign(1, 0);

    uint64_t N[3] = {0, 0, 0}, nHits = 0, nMulti = 0, nIsoMulti = 0, cnt = 0;
    std::map<int, uint64_t> counter;   // #alignments of a read -> #reads (the histogram at the end of .cnt)
    Read read, record_read;
    Hit hit{0, 0, 0};
    std::vector<Hit> hits;
    std::vector<int> gids;
    char tmp[64];

    auto write_read = [&](const Read& r, int category) {   // SingleRead(Q)::write, PairedEndRead(Q)::write
        for (int m = 0; m < n_os; ++m) {
            OutFile& o = cat[category][m];
            o.put(ps.hasq ? '@' : '>');
            o.put(r.mate[m].name);
            o.put('\n');
            o.put(r.mate[m].seq);
            o.put('\n');
            if (ps.hasq) { o.put("+\n", 2); o.put(r.mate[m].qual); o.put('\n'); }
        }
        append_read(sc.reads[category], sc.shorts[category], r, n_os, ps.hasq);
        ++N[category];
    };
    auto flush_hits = [&]() {   // one line of .dat + the statistics of parseIt.cpp:88-103
        const size_t k = hits.size();
        nHits += k;
        gids.clear();
        for (const Hit& h : hits) gids.push_back(gid[(size_t)std::abs(h.sid)]);
        std::sort(gids.begin(), gids.end());
        if (std::unique(gids.begin(), gids.end()) - gids.begin() > 1) ++nMulti;
        if (k > 1) ++nIsoMulti;
        dat.put(tmp, (size_t)(put_int(tmp, (long long)k) - tmp));
        for (const Hit& h : hits) {
            char* e = tmp;
            *e++ = ' '; e = put_int(e, h.sid);
            *e++ = ' '; e = put_int(e, h.pos);
            if (ps.paired) { *e++ = ' '; e = put_int(e, h.insertL); }
            dat.put(tmp, (size_t)(e - tmp));
            sc.hits.sid.push_back(h.sid);
            sc.hits.pos.push_back(h.pos);
            if (ps.paired) sc.hits.insertL.push_back(h.insertL);
        }
        dat.put('\n');
        sc.hits.row_ptr.push_back(sc.hits.sid.size());
        ++counter[(int)k];
    };

    int val, record_val = -2;   // -2: no read recorded yet
    while ((val = ps.next(read, hit)) >= 0) {
        if (val <= 2) {
            if (record_val >= 0) write_read(record_read, record_val);
            if (!(record_val == 1 || hits.empty()))
                die("Read " + record_read.name + " is both unalignable and alignable according to the input file!");
            if (record_val == 1) flush_hits();
            hits.clear();
            record_val = val;
            record_read = read;
        }
        if (val == 1 || val == 5) hits.push_back(hit);
        ++cnt;
        if (g_verbose && cnt % 1000000 == 0) { printf("Parsed %llu entries\n", (unsigned long long)cnt); fflush(stdout); }
    }
    if (record_val >= 0) write_read(record_read, record_val);
    if (record_val == 1) flush_hits();
    if (ps.n_warns > 0) fprintf(stderr, "Warning: Detected %d lines containing read pairs whose two mates have different names.\n", ps.n_warns);
    const uint64_t nUnique = N[1] - nMulti;

    dat.flush();
    for (int t = 0; t < 3; ++t) for (int m = 0; m < n_os; ++m) cat[t][m].flush();
    writer.drain();
    {   // the header over the reserved blanks
        const int n = snprintf(tmp, sizeof tmp, "%llu %llu %d", (unsigned long long)N[1], (unsigned long long)nHits, read_type);
        if (fseek(dat.f, 0, SEEK_SET) != 0 || fwrite(tmp, 1, (size_t)n, dat.f) != (size_t)n) die("Cannot write " + dat.path + "!");
    }
    dat.close();

    {   // statName.cnt (parseIt.cpp:213-223)
        FILE* fo = fopen((statName + ".cnt").c_str(), "w");
        if (!fo) die("Cannot open " + statName + ".cnt for writing!");
        fprintf(fo, "%llu %llu %llu %llu\n", (unsigned long long)N[0], (unsigned long long)N[1], (unsigned long long)N[2],
                (unsigned long long)(N[0] + N[1] + N[2]));
        fprintf(fo, "%llu %llu %llu\n", (unsigned long long)nUnique, (unsigned long long)nMulti, (unsigned long long)nIsoMulti);
        fprintf(fo, "%llu %d\n", (unsigned long long)nHits, read_type);
        fprintf(fo, "0\t%llu\n", (unsigned long long)N[0]);
        for (const auto& kv : counter) fprintf(fo, "%d\t%llu\n", kv.first, (unsigned long long)kv.second);
        fprintf(fo, "Inf\t%llu\n", (unsigned long long)N[2]);
        fclose(fo);
    }

    for (int t = 0; t < 3; ++t)
        for (int m = 0; m < n_os; ++m) {
            cat[t][m].close();
            if (N[t] == 0) remove(cat[t][m].path.c_str());   // empty categories leave no file
        }

    if (sidecar_enabled()) {
        sc.hits.N = N[1];
        sc.hits.H = nHits;
        write_sidecar(imdName, sc);
    }
    if (g_verbose) printf("Done!\n");
    return 0;
}
