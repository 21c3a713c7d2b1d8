// Parsers for the reference's intermediate files.  All of them work on a whole-file buffer with a
// hand-rolled tokenizer (the reference uses istream >>, 6e6 hits/s; see SURVEY.md section 8(f).2).
#include <sys/stat.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <set>
#include <thread>

#include "host.hpp"

namespace host {

bool g_verbose = true;
int g_io_threads = 1;

void parallel_ranges(size_t n, int parts, const std::function<void(size_t, size_t, int)>& fn) {
    if (parts < 1) parts = 1;
    if ((size_t)parts > n) parts = n ? (int)n : 1;
    if (parts == 1) { fn(0, n, 0); return; }
    std::vector<std::thread> pool;
    for (int t = 0; t < parts; ++t) {
        const size_t b = n * (size_t)t / parts, e = n * (size_t)(t + 1) / parts;
        pool.emplace_back([&fn, b, e, t]() { fn(b, e, t); });
    }
    for (auto& th : pool) th.join();
}

void die(const std::string& msg) {
    fprintf(stderr, "%s\n", msg.c_str());
    exit(-1);
}

void check_rc(int rc, const char* what) {
    if (rc != 0) die(std::string("rsem_b200: ") + what + " failed: " + rsem_b200_last_error());
}

std::vector<char> slurp(const std::string& path, bool must_exist) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) {
        if (must_exist) die("Cannot open " + path + "! It may not exist.");
        return {};
    }
    struct stat st;
    std::vector<char> buf;
    if (fstat(fileno(f), &st) == 0 && st.st_size > 0) {
        buf.resize((size_t)st.st_size);
        size_t got = fread(buf.data(), 1, buf.size(), f);
        buf.resize(got);
    }
    fclose(f);
    return buf;
}

std::vector<uint32_t> engine_seeds(uint32_t seed, int n) {
    Mt seedEngine(seed);
    std::set<uint32_t> used;
    std::vector<uint32_t> out(n);
    for (int i = 0; i < n; ++i) {
        uint32_t s;
        do { s = seedEngine.next(); } while (used.count(s));
        used.insert(s);
        out[i] = s;
    }
    return out;
}

uint32_t parse_seed(const char* s) {
    uint32_t seed = 0;
    for (const char* p = s; *p; ++p) seed = seed * 10 + (uint32_t)(*p - '0');
    return seed;
}

std::vector<int> gpu_devices() {
    std::vector<int> devices;
    if (const char* e = getenv("RSEM_B200_DEVICES")) {  // e.g. "0,1,2,3"
        for (const char* q = e; *q;) {
            devices.push_back(atoi(q));
            while (*q && *q != ',') ++q;
            if (*q == ',') ++q;
        }
    }
    if (devices.size() <= 1) {
        const char* one = getenv("RSEM_B200_DEVICE");
        devices.assign(1, one ? atoi(one) : devices.empty() ? 0 : devices[0]);
    }
    return devices;
}

namespace {

struct Cursor {
    const char* p;
    const char* end;
    explicit Cursor(const std::vector<char>& b) : p(b.data()), end(b.data() + b.size()) {}
    void skip_ws() { while (p < end && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) ++p; }
    bool eof() { skip_ws(); return p >= end; }
    bool next_i64(long long& v) {
        skip_ws();
        if (p >= end) return false;
        bool neg = false;
        if (*p == '-') { neg = true; ++p; } else if (*p == '+') ++p;
        if (p >= end || *p < '0' || *p > '9') return false;
        long long x = 0;
        while (p < end && *p >= '0' && *p <= '9') x = x * 10 + (*p++ - '0');
        v = neg ? -x : x;
        return true;
    }
    bool next_f64(double& v) {
        skip_ws();
        if (p >= end) return false;
        char tmp[64];
        size_t n = 0;
        while (p + n < end && n < 63 && !(p[n] == ' ' || p[n] == '\n' || p[n] == '\t' || p[n] == '\r')) { tmp[n] = p[n]; ++n; }
        tmp[n] = 0;
        char* e = nullptr;
        v = strtod(tmp, &e);
        if (e == tmp) return false;
        p += (e - tmp);
        return true;
    }
    // rest of the current line (without the newline); false at EOF
    bool line(const char*& b, size_t& n) {
        if (p >= end) return false;
        b = p;
        const char* q = (const char*)memchr(p, '\n', (size_t)(end - p));
        if (!q) { n = (size_t)(end - p); p = end; }
        else { n = (size_t)(q - p); p = q + 1; }
        return true;
    }
};

int8_t g_code[256];
bool g_code_init = false;
void init_codes() {
    if (g_code_init) return;
    memset(g_code, -1, sizeof g_code);
    g_code[(int)'a'] = g_code[(int)'A'] = 0;
    g_code[(int)'c'] = g_code[(int)'C'] = 1;
    g_code[(int)'g'] = g_code[(int)'G'] = 2;
    g_code[(int)'t'] = g_code[(int)'T'] = 3;
    g_code[(int)'n'] = g_code[(int)'N'] = 4;
    g_code_init = true;
}

}  // namespace

// ---- ref.seq ------------------------------------------------------------------------------------
void load_refs(const std::string& path, bool with_seqs, RefData& r) {
    init_codes();
    std::vector<char> buf = slurp(path);
    Cursor c(buf);
    r = RefData();
    r.seq_off.push_back(0);
    r.full_len.push_back(0);
    r.tot_len.push_back(0);
    r.mask_off.push_back(0);
    long long fullLen, totLen;
    while (c.next_i64(fullLen)) {
        if (!c.next_i64(totLen)) break;
        const char* b; size_t n;
        c.line(b, n);                      // rest of the length line
        if (!c.line(b, n)) break;          // name
        if (!c.line(b, n)) break;          // sequence
        if (fullLen <= 0 || totLen < fullLen) die("Corrupted reference file " + path);
        r.seq_off.push_back(r.seq.size());
        if (with_seqs) {
            if ((long long)n < totLen) die("Reference sequence shorter than its declared length in " + path);
            size_t at = r.seq.size();
            r.seq.resize(at + (size_t)totLen);
            for (long long k = 0; k < totLen; ++k) {
                int8_t code = g_code[(unsigned char)b[k]];
                if (code < 0) {
                    fprintf(stderr, "Found unknown sequence letter %c at function get_base_id!\n", b[k]);
                    exit(-1);
                }
                r.seq[at + k] = (uint8_t)code;
            }
        }
        r.full_len.push_back((int32_t)fullLen);
        r.tot_len.push_back((int32_t)totLen);
        r.mask_off.push_back(r.mask_words.size());
        const int nw = (int)((fullLen - 1) / 32 + 1);
        for (int k = 0; k < nw; ++k) {
            long long w;
            if (!c.next_i64(w)) die("Corrupted mask words in " + path);
            r.mask_words.push_back((uint32_t)w);
        }
        c.line(b, n);  // end of the mask line
        ++r.M;
        r.has_polyA = r.has_polyA || fullLen < totLen;
    }
    r.seq_off.push_back(r.seq.size());
    if (g_verbose) printf("Refs.loadRefs finished!\n");
}

// ---- ref.ti ---------------------------------------------------------------------------------------
void load_transcripts(const std::string& path, std::vector<TranscriptInfo>& out, int* type_out) {
    std::ifstream fin(path.c_str());
    if (!fin.is_open()) { fprintf(stderr, "Cannot open %s! It may not exist.\n", path.c_str()); exit(-1); }
    int M, type;
    std::string line;
    fin >> M >> type;
    if (type_out) *type_out = type;
    getline(fin, line);
    out.assign(M + 1, TranscriptInfo());
    for (int i = 1; i <= M; ++i) {
        TranscriptInfo& t = out[i];
        getline(fin, line);
        size_t tab = line.find('\t');
        t.transcript_id = line.substr(0, tab);
        t.transcript_name = tab == std::string::npos ? "" : line.substr(tab + 1);
        getline(fin, line);
        tab = line.find('\t');
        t.gene_id = line.substr(0, tab);
        t.gene_name = tab == std::string::npos ? "" : line.substr(tab + 1);
        getline(fin, t.seqname);
        std::string strand;
        int s;
        fin >> strand >> t.length >> s;
        t.strand = strand.empty() ? '+' : strand[0];
        for (int k = 0; k < s; ++k) {
            int a, b;
            fin >> a >> b;
            t.exons.emplace_back(a, b);
            t.exon_length += b - a + 1;
        }
        getline(fin, line);
        getline(fin, line);  // "left"
    }
}

std::vector<int> map_bam_targets(const std::vector<std::string>& names, const std::vector<TranscriptInfo>& tr, int ti_type) {
    const int M = (int)tr.size() - 1;
    if (names.empty()) die("The SAM/BAM file declares less than one reference sequence!");
    if ((int)names.size() > M) die("The SAM/BAM file declares more reference sequences (" + std::to_string(names.size()) + ") than RSEM knows (" + std::to_string(M) + ")!");
    if ((int)names.size() < M)
        fprintf(stderr, "Warning: The SAM/BAM file declares less reference sequences (%d) than RSEM knows (%d)! Please make sure that you aligned your reads against transcript sequences instead of genome.\n", (int)names.size(), M);
    std::map<std::string, int> dict;
    for (int i = 1; i <= M; ++i) {
        const std::string& tid = ti_type == 2 ? tr[i].seqname : tr[i].transcript_id;
        if (!dict.emplace(tid, i).second) die("RSEM's indices might be corrupted, " + tid + " appears more than once!");
    }
    std::vector<int> e2i(names.size(), 0);
    for (size_t i = 0; i < names.size(); ++i) {
        auto it = dict.find(names[i]);
        if (it == dict.end()) die("RSEM can not recognize reference sequence name " + names[i] + "!");
        if (it->second < 0) die("Reference sequence name " + names[i] + " appears more than once in the SAM/BAM file!");
        e2i[i] = it->second;
        it->second = -1;
    }
    return e2i;
}

void load_groups(const std::string& path, std::vector<int>& starts) {
    FILE* fi = fopen(path.c_str(), "r");
    if (!fi) { fprintf(stderr, "Cannot open %s! It may not exist.\n", path.c_str()); exit(-1); }
    starts.clear();
    int pos;
    while (fscanf(fi, "%d", &pos) == 1) starts.push_back(pos);
    fclose(fi);
}

bool load_allele_groups(const std::string& ref_name, std::vector<int>& gt, std::vector<int>& ta) {
    FILE* a = fopen((ref_name + ".gt").c_str(), "r");
    FILE* b = fopen((ref_name + ".ta").c_str(), "r");
    const bool ok = a && b;
    if (a) fclose(a);
    if (b) fclose(b);
    if (ok) { load_groups(ref_name + ".gt", gt); load_groups(ref_name + ".ta", ta); }
    return ok;
}

void load_mparams(const std::string& path, ModelParamsH& p) {
    std::vector<char> buf = slurp(path);
    Cursor c(buf);
    long long v = 0;
    double d = 0.0;
    bool ok = c.next_i64(v); p.minL = (int)v;
    ok = ok && c.next_i64(v); p.maxL = (int)v;
    ok = ok && c.next_f64(d); p.probF = d;
    ok = ok && c.next_i64(v); p.estRSPD = v != 0;
    ok = ok && c.next_i64(v); p.B = (int)v;
    ok = ok && c.next_i64(v); p.mate_minL = (int)v;
    ok = ok && c.next_i64(v); p.mate_maxL = (int)v;
    ok = ok && c.next_f64(d); p.mean = d;
    ok = ok && c.next_f64(d); p.sd = d;
    ok = ok && c.next_i64(v); p.seedLen = (int)v;
    if (!ok) die("Cannot parse " + path + "!");
}

// ---- reads ----------------------------------------------------------------------------------------
void read_type_files(const std::string& imd, int tag, int read_type, std::vector<std::string>& files) {
    static const char* tags[3] = {"un", "alignable", "max"};
    const char* suffix = (read_type == 0 || read_type == 2) ? "fa" : "fq";
    files.clear();
    if (read_type < 2) files.push_back(imd + "_" + tags[tag] + "." + suffix);
    else {
        files.push_back(imd + "_" + tags[tag] + "_1." + suffix);
        files.push_back(imd + "_" + tags[tag] + "_2." + suffix);
    }
}

namespace {
// SingleRead(Q)::calc_lq, SingleReadQ.h:63-95
bool single_lq(const char* s, int len, bool has_polyA, int seed_len) {
    if (len < seed_len) return true;
    if (!has_polyA) return false;
    int numA = 0, numT = 0, numAO = 0, numTO = 0;
    const int threshold_1 = int(0.9 * len - 1.5 * sqrt(len * 1.0) + 0.5);
    const int threshold_2 = (kOlen - 1) / 2 + 1;
    for (int i = 0; i < len; ++i) {
        if (s[i] == 'A') { ++numA; if (i < kOlen) ++numAO; }
        if (s[i] == 'T') { ++numT; if (i >= len - kOlen) ++numTO; }
    }
    if (numA >= threshold_1) return numAO >= threshold_2;
    if (numT >= threshold_1) return numTO >= threshold_2;
    return false;
}
}  // namespace

// Whole read set -> ReadStore, split over g_io_threads:
//   1. newline index of every file (per-chunk counts, prefix sum, fill);
//   2. a record is 4 (FASTQ) / 2 (FASTA) lines; lengths -> offsets by prefix sum;
//   3. records converted in parallel straight into their final slots.
// `short_names` receives the first 50 names of reads dropped for length < seed length (the reference warns about
// those), `n_short` their total number.
void parse_reads(const std::string& imd, int tag, int read_type, bool has_polyA, int seed_len, ReadStore& out,
                 std::vector<std::string>* short_names, uint64_t* n_short) {
    init_codes();
    const int s = read_type >= 2 ? 2 : 1;
    const bool hasq = read_type & 1;
    const int lpr = hasq ? 4 : 2;
    std::vector<std::string> files;
    read_type_files(imd, tag, read_type, files);
    std::vector<char> buf[2];
    for (int m = 0; m < s; ++m) {
        FILE* f = fopen(files[m].c_str(), "rb");
        if (!f) { fprintf(stderr, "Cannot open %s! It may not exist.\n", files[m].c_str()); exit(-1); }
        fclose(f);
        buf[m] = slurp(files[m]);
        if (!buf[m].empty() && buf[m].back() != '\n') buf[m].push_back('\n');
    }
    // line starts
    std::vector<size_t> line[2];
    for (int m = 0; m < s; ++m) {
        const char* base = buf[m].data();
        const size_t n = buf[m].size();
        const int T = std::max(1, std::min(g_io_threads, (int)(n >> 20) + 1));
        std::vector<size_t> cnt(T + 1, 0);
        parallel_ranges(n, T, [&](size_t b, size_t e, int t) {
            size_t c = 0;
            for (const char* q = base + b; (q = (const char*)memchr(q, '\n', (size_t)(base + e - q))) != nullptr; ++q) ++c;
            cnt[t + 1] = c;
        });
        for (int t = 0; t < T; ++t) cnt[t + 1] += cnt[t];
        line[m].resize(cnt[T] + 1);
        line[m][0] = 0;
        parallel_ranges(n, T, [&](size_t b, size_t e, int t) {
            size_t at = cnt[t] + 1;
            for (const char* q = base + b; (q = (const char*)memchr(q, '\n', (size_t)(base + e - q))) != nullptr; ++q)
                line[m][at++] = (size_t)(q - base) + 1;
        });
    }
    uint64_t n_rec = (line[0].size() - 1) / lpr;
    if (s == 2) n_rec = std::min<uint64_t>(n_rec, (line[1].size() - 1) / lpr);
    out = ReadStore();
    out.n_mates = s;
    out.has_qual = hasq;
    out.n = n_rec;
    out.lowq.assign(n_rec, 0);
    auto seq_of = [&](int m, uint64_t r, const char*& p, int& len) {
        const size_t a = line[m][r * lpr + 1], b = line[m][r * lpr + 2];
        p = buf[m].data() + a;
        len = (int)(b - a - 1);
        while (len > 0 && p[len - 1] == '\r') --len;
    };
    for (int m = 0; m < s; ++m) {
        out.off[m].assign(n_rec + 1, 0);
        parallel_ranges((size_t)n_rec, g_io_threads, [&](size_t b, size_t e, int) {
            for (size_t r = b; r < e; ++r) { const char* p; int len; seq_of(m, r, p, len); out.off[m][r + 1] = (uint64_t)len; }
        });
        for (uint64_t r = 0; r < n_rec; ++r) out.off[m][r + 1] += out.off[m][r];
        out.base[m].resize(out.off[m][n_rec]);
        if (hasq) out.qual[m].resize(out.off[m][n_rec]);
    }
    const int T = std::max(1, std::min<int>(g_io_threads, (int)(n_rec / 4096) + 1));
    std::vector<std::vector<std::string>> shorts(T);
    std::vector<uint64_t> short_cnt(T, 0);
    std::vector<std::string> errors(T);
    parallel_ranges((size_t)n_rec, T, [&](size_t rb, size_t re, int t) {
        for (size_t r = rb; r < re; ++r) {
            const char* sp[2] = {nullptr, nullptr};
            int len[2] = {0, 0};
            for (int m = 0; m < s; ++m) {
                const char* hdr = buf[m].data() + line[m][r * lpr];
                if (*hdr != (hasq ? '@' : '>')) { errors[t] = hasq ? "Read file does not look like a FASTQ file!" : "Read file does not look like a FASTA file!"; return; }
                seq_of(m, r, sp[m], len[m]);
                if (hasq && buf[m][line[m][r * lpr + 2]] != '+') { errors[t] = "Read file does not look like a FASTQ file!"; return; }
            }
            bool lq;
            if (s == 1) lq = seed_len > 0 ? single_lq(sp[0], len[0], has_polyA, seed_len) : false;
            else if (seed_len <= 0) lq = false;
            else if (len[0] < seed_len || len[1] < seed_len) lq = true;  // PairedEndReadQ.h:58-65
            else lq = single_lq(sp[0], len[0], has_polyA, seed_len) && single_lq(sp[1], len[1], has_polyA, seed_len);
            out.lowq[r] = lq ? 1 : 0;
            if (lq && short_names && (s == 1 ? len[0] < seed_len : (len[0] < seed_len || len[1] < seed_len))) {
                const char* hdr = buf[0].data() + line[0][r * lpr];
                size_t hl = line[0][r * lpr + 1] - line[0][r * lpr] - 1;
                ++short_cnt[t];
                if (shorts[t].size() < 50) shorts[t].emplace_back(hdr + 1, hl ? hl - 1 : 0);
            }
            for (int m = 0; m < s; ++m) {
                uint8_t* bd = out.base[m].data() + out.off[m][r];
                for (int k = 0; k < len[m]; ++k) {
                    int8_t code = g_code[(unsigned char)sp[m][k]];
                    if (code < 0) {
                        if (!lq) { errors[t] = std::string("Found unknown sequence letter ") + sp[m][k] + " at function get_base_id!"; return; }
                        code = 4;
                    }
                    bd[k] = (uint8_t)code;
                }
                if (hasq) {
                    const size_t qa = line[m][r * lpr + 3];
                    int ql = (int)(line[m][r * lpr + 4] - qa - 1);
                    const char* qp = buf[m].data() + qa;
                    while (ql > 0 && qp[ql - 1] == '\r') --ql;
                    if (ql != len[m]) { errors[t] = "A read has a different number of bases and quality values!"; return; }
                    uint8_t* qd = out.qual[m].data() + out.off[m][r];
                    for (int k = 0; k < len[m]; ++k) {
                        const int q = (unsigned char)qp[k];
                        if (q < 33 || q > 126) { errors[t] = "A read has a quality character outside [33, 126]!"; return; }
                        qd[k] = (uint8_t)(q - 33);
                    }
                }
            }
        }
    });
    for (const std::string& e : errors) if (!e.empty()) die(e);
    if (short_names)
        for (auto& v : shorts) for (auto& nm : v) if (short_names->size() < 50) short_names->push_back(nm);
    if (n_short) { *n_short = 0; for (uint64_t c : short_cnt) *n_short += c; }
}

// ---- imd.dat --------------------------------------------------------------------------------------
// The body is one line per read: the buffer is cut at newlines into one piece per thread, every piece is tokenised into
// its own arrays and the pieces are concatenated.
void load_dat(const std::string& path, int read_type, uint64_t expect_n1, HitStore& h) {
    std::vector<char> buf = slurp(path);
    Cursor c(buf);
    long long n1, nh, rt;
    if (!c.next_i64(n1) || !c.next_i64(nh) || !c.next_i64(rt)) die("Cannot read alignments from .dat file!");
    if ((uint64_t)n1 != expect_n1) die("Number of alignable reads does not match!");
    if (rt != read_type) die("Data file (.dat) does not have the right read type!");
    const bool paired = read_type >= 2;
    const char* body = c.p;
    const char* end = buf.data() + buf.size();
    const int T = std::max(1, std::min(g_io_threads, (int)((end - body) / (1 << 20)) + 1));
    std::vector<const char*> cut(T + 1);
    cut[0] = body;
    cut[T] = end;
    for (int t = 1; t < T; ++t) {
        const char* q = body + (size_t)(end - body) * t / T;
        const char* nl = (const char*)memchr(q, '\n', (size_t)(end - q));
        cut[t] = nl ? nl + 1 : end;
    }
    struct Piece { std::vector<uint64_t> deg; std::vector<int32_t> sid, pos, ins; bool bad = false; };
    std::vector<Piece> pieces(T);
    parallel_ranges((size_t)T, T, [&](size_t b, size_t, int) {
        Piece& pc = pieces[b];
        Cursor cur(buf);
        cur.p = cut[b];
        cur.end = cut[b + 1];
        long long k, x, y, l = 0;
        while (cur.next_i64(k)) {
            if (k <= 0) { pc.bad = true; return; }
            for (long long j = 0; j < k; ++j) {
                if (!cur.next_i64(x) || !cur.next_i64(y) || (paired && !cur.next_i64(l))) { pc.bad = true; return; }
                pc.sid.push_back((int32_t)x);
                pc.pos.push_back((int32_t)y);
                if (paired) pc.ins.push_back((int32_t)l);
            }
            pc.deg.push_back((uint64_t)k);
        }
    });
    uint64_t N = 0, H = 0;
    for (auto& pc : pieces) {
        if (pc.bad) die("Cannot read alignments from .dat file!");
        N += pc.deg.size();
        H += pc.sid.size();
    }
    if (N != (uint64_t)n1) die("Cannot read alignments from .dat file!");
    h.N = N;
    h.H = H;
    h.row_ptr.resize(N + 1);
    h.sid.resize(H);
    h.pos.resize(H);
    h.insertL.resize(paired ? H : 0);
    std::vector<uint64_t> n_off(T + 1, 0), h_off(T + 1, 0);
    for (int t = 0; t < T; ++t) { n_off[t + 1] = n_off[t] + pieces[t].deg.size(); h_off[t + 1] = h_off[t] + pieces[t].sid.size(); }
    parallel_ranges((size_t)T, T, [&](size_t b, size_t, int) {
        const Piece& pc = pieces[b];
        uint64_t at = h_off[b];
        for (size_t i = 0; i < pc.deg.size(); ++i) { h.row_ptr[n_off[b] + i] = at; at += pc.deg[i]; }
        if (!pc.sid.empty()) {
            memcpy(h.sid.data() + h_off[b], pc.sid.data(), pc.sid.size() * sizeof(int32_t));
            memcpy(h.pos.data() + h_off[b], pc.pos.data(), pc.pos.size() * sizeof(int32_t));
            if (paired) memcpy(h.insertL.data() + h_off[b], pc.ins.data(), pc.ins.size() * sizeof(int32_t));
        }
    });
    h.row_ptr[N] = H;
}

// ---- imd.ofg ---------------------------------------------------------------------------------------
namespace {
// Binary side-car of imd.ofg (SURVEY 8(f).2): the rows rsem-run-gibbs would parse from the text, in upload layout.  The values
// are the doubles the TEXT denotes (15 significant digits, parsed back with strtod while the line is formatted), not the
// unrounded conprb: the Gibbs draws must be the ones the reference makes from the text file.
struct OfgHeader {
    char magic[8];      // "RSEMOFG1"
    uint64_t M, N0, rows, entries, ofg_bytes;
};
const char kOfgMagic[8] = {'R', 'S', 'E', 'M', 'O', 'F', 'G', '1'};

uint64_t file_size_of(const std::string& path) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return 0;
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fclose(f);
    return n < 0 ? 0 : (uint64_t)n;
}
}  // namespace

void write_ofg(const std::string& path, int M, uint64_t N0, const HitStore& h, const std::vector<double>& conprb,
               const std::vector<double>& ncpv) {
    FILE* fo = fopen(path.c_str(), "w");
    if (!fo) die("Cannot open " + path + " for writing!");
    fprintf(fo, "%d %llu\n", M, (unsigned long long)N0);
    const bool side = sidecar_enabled();
    const int T = std::max(1, std::min<int>(g_io_threads, (int)(h.H / 200000) + 1));
    std::vector<std::string> text(T);
    struct Bin { std::vector<uint32_t> deg; std::vector<int32_t> sid; std::vector<double> val; };
    std::vector<Bin> bin(T);
    parallel_ranges((size_t)h.N, T, [&](size_t b, size_t e, int t) {   // "%.15g" like ostream << setprecision(15)
        std::string& out = text[t];
        Bin& bn = bin[t];
        out.reserve((size_t)((h.row_ptr[e] - h.row_ptr[b]) * 26 + (e - b) * 24));
        if (side) { bn.sid.reserve((size_t)(h.row_ptr[e] - h.row_ptr[b]) + (e - b)); bn.val.reserve(bn.sid.capacity()); bn.deg.reserve(e - b); }
        char tmp[64];
        auto emit = [&](int id, double v) {
            const int n = snprintf(tmp, sizeof tmp, "%d %.15g ", id, v);
            out.append(tmp, (size_t)n);
            if (side) { bn.sid.push_back(id); bn.val.push_back(strtod(strchr(tmp, ' ') + 1, nullptr)); }
        };
        for (size_t i = b; i < e; ++i) {
            uint32_t tot = 0;
            if (ncpv[i] >= kEps) { ++tot; emit(0, ncpv[i]); }
            for (uint64_t j = h.row_ptr[i]; j < h.row_ptr[i + 1]; ++j)
                if (conprb[j] >= kEps) { ++tot; emit(abs(h.sid[j]), conprb[j]); }
            if (tot > 0) { out.push_back('\n'); if (side) bn.deg.push_back(tot); }
        }
    });
    for (const std::string& piece : text) fwrite(piece.data(), 1, piece.size(), fo);
    if (fclose(fo) != 0) die("Cannot write " + path + " (disk full?)!");
    if (!side) return;
    OfgHeader hd;
    memset(&hd, 0, sizeof hd);
    memcpy(hd.magic, kOfgMagic, 8);
    hd.M = (uint64_t)M;
    hd.N0 = N0;
    for (const Bin& bn : bin) { hd.rows += bn.deg.size(); hd.entries += bn.sid.size(); }
    hd.ofg_bytes = file_size_of(path);
    std::vector<uint64_t> row_ptr;
    row_ptr.reserve((size_t)hd.rows + 1);
    uint64_t at = 0;
    row_ptr.push_back(0);
    for (const Bin& bn : bin) for (uint32_t d : bn.deg) { at += d; row_ptr.push_back(at); }
    FILE* fb = fopen((path + ".b200").c_str(), "wb");
    if (!fb) die("Cannot open " + path + ".b200 for writing!");
    bool ok = fwrite(&hd, sizeof hd, 1, fb) == 1 && fwrite(row_ptr.data(), 8, row_ptr.size(), fb) == row_ptr.size();
    for (const Bin& bn : bin) ok = ok && (bn.sid.empty() || fwrite(bn.sid.data(), 4, bn.sid.size(), fb) == bn.sid.size());
    for (const Bin& bn : bin) ok = ok && (bn.val.empty() || fwrite(bn.val.data(), 8, bn.val.size(), fb) == bn.val.size());
    if (fclose(fb) != 0 || !ok) die("Cannot write " + path + ".b200 (disk full?)!");
}

// the side-car of `path`, if it is present and still describes the text file next to it
static bool load_ofg_sidecar(const std::string& path, int M, uint64_t& N0, std::vector<uint64_t>& row_ptr, std::vector<int32_t>& sid,
                             std::vector<double>& conprb) {
    if (!sidecar_enabled()) return false;
    FILE* fb = fopen((path + ".b200").c_str(), "rb");
    if (!fb) return false;
    OfgHeader hd;
    const uint64_t have = file_size_of(path + ".b200");
    bool ok = fread(&hd, sizeof hd, 1, fb) == 1 && !memcmp(hd.magic, kOfgMagic, 8) && hd.M == (uint64_t)M &&
              hd.ofg_bytes == file_size_of(path) && hd.ofg_bytes > 0 && hd.entries <= have / 12 && hd.rows <= have / 8 &&
              have == sizeof hd + 8 * (hd.rows + 1) + 12 * hd.entries;
    if (ok) {
        row_ptr.resize((size_t)hd.rows + 1);
        sid.resize((size_t)hd.entries);
        conprb.resize((size_t)hd.entries);
        ok = fread(row_ptr.data(), 8, row_ptr.size(), fb) == row_ptr.size() &&
             (hd.entries == 0 || (fread(sid.data(), 4, sid.size(), fb) == sid.size() && fread(conprb.data(), 8, conprb.size(), fb) == conprb.size())) &&
             row_ptr[0] == 0 && row_ptr[(size_t)hd.rows] == hd.entries;
        N0 = hd.N0;
    }
    fclose(fb);
    return ok;
}

void load_ofg(const std::string& path, int M, uint64_t& N0, std::vector<uint64_t>& row_ptr, std::vector<int32_t>& sid,
              std::vector<double>& conprb, bool allow_sidecar) {
    if (allow_sidecar && load_ofg_sidecar(path, M, N0, row_ptr, sid, conprb)) return;
    std::vector<char> buf = slurp(path, false);
    if (buf.empty()) die("Cannot open " + path + "!");
    if (buf.back() != '\n') buf.push_back('\n');
    buf.push_back('\0');
    const char* p = buf.data();
    const char* end = p + buf.size() - 1;
    char* q = nullptr;
    const long long m = strtoll(p, &q, 10);
    p = q;
    N0 = strtoull(p, &q, 10);
    p = q;
    if (m != M) die("M in " + path + " is not consistent with the reference!");
    while (p < end && *p != '\n') ++p;
    ++p;
    const char* body = p;
    const int T = std::max(1, std::min(g_io_threads, (int)((end - body) / (1 << 20)) + 1));
    std::vector<const char*> cut(T + 1);
    cut[0] = body;
    cut[T] = end;
    for (int t = 1; t < T; ++t) {
        const char* s0 = body + (size_t)(end - body) * t / T;
        const char* nl = (const char*)memchr(s0, '\n', (size_t)(end - s0));
        cut[t] = nl ? nl + 1 : end;
    }
    struct Piece { std::vector<uint64_t> deg; std::vector<int32_t> sid; std::vector<double> val; };
    std::vector<Piece> pieces(T);
    parallel_ranges((size_t)T, T, [&](size_t b, size_t, int) {   // one row per line (Gibbs.cpp:121-134), empty lines count too
        Piece& pc = pieces[b];
        const char* s0 = cut[b];
        const char* e0 = cut[b + 1];
        while (s0 < e0) {
            const char* eol = (const char*)memchr(s0, '\n', (size_t)(e0 - s0));
            if (!eol) eol = e0;
            uint64_t n = 0;
            while (s0 < eol) {
                while (s0 < eol && (*s0 == ' ' || *s0 == '\t' || *s0 == '\r')) ++s0;
                if (s0 >= eol) break;
                char* r = nullptr;
                const long id = strtol(s0, &r, 10);
                if (r == s0) break;
                s0 = r;
                const double v = strtod(s0, &r);
                if (r == s0) break;
                s0 = r;
                pc.sid.push_back((int32_t)id);
                pc.val.push_back(v);
                ++n;
            }
            pc.deg.push_back(n);
            s0 = eol + 1;
        }
    });
    uint64_t N = 0, E = 0;
    std::vector<uint64_t> n_off(T + 1, 0), e_off(T + 1, 0);
    for (int t = 0; t < T; ++t) {
        n_off[t + 1] = n_off[t] + pieces[t].deg.size();
        e_off[t + 1] = e_off[t] + pieces[t].sid.size();
    }
    N = n_off[T];
    E = e_off[T];
    row_ptr.resize(N + 1);
    sid.resize(E);
    conprb.resize(E);
    parallel_ranges((size_t)T, T, [&](size_t b, size_t, int) {
        const Piece& pc = pieces[b];
        uint64_t at = e_off[b];
        for (size_t i = 0; i < pc.deg.size(); ++i) { row_ptr[n_off[b] + i] = at; at += pc.deg[i]; }
        if (!pc.sid.empty()) {
            memcpy(sid.data() + e_off[b], pc.sid.data(), pc.sid.size() * sizeof(int32_t));
            memcpy(conprb.data() + e_off[b], pc.val.data(), pc.val.size() * sizeof(double));
        }
    });
    row_ptr[N] = E;
}

}  // namespace host
