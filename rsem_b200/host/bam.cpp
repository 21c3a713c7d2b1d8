// SAM / BAM input and BAM output for rsem-run-em -b (posterior-annotated transcript BAM).
//
// What it replaces: the reference re-reads its input alignment file with htslib and writes every record back with
// MAPQ and a ZW:f tag set from the posterior of the alignment (/root/reference/BamWriter.h:39-48, 82-146;
// sam_utils.h:72-76), in input order.  The reference vendors htslib for this; here the two container formats are
// implemented directly on zlib (SAM v1 / BAM as in the SAM specification, BGZF = concatenated gzip members with a
// "BC" extra field), because only sequential record read / rewrite is needed:
//   * AlnReader: SAM text (plain or gzip) or BAM; yields BAM-encoded records (SAM lines are converted with the same
//     field encodings htslib's sam_parse1 uses, e.g. the smallest integer type for i-tags);
//   * BamWriter: BGZF blocks of <= 0xff00 bytes, compressed by a pool of host threads (-p), written in order, EOF marker.
// CRAM is not supported (the run stops with a clear message).
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <thread>

#include "host.hpp"

namespace host {

namespace {

inline uint32_t rd_u32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
inline uint16_t rd_u16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }
inline void wr_u32(uint8_t* p, uint32_t v) { p[0] = v & 255; p[1] = (v >> 8) & 255; p[2] = (v >> 16) & 255; p[3] = (v >> 24) & 255; }
inline void wr_u16(uint8_t* p, uint16_t v) { p[0] = v & 255; p[1] = (v >> 8) & 255; }
template <class T>
inline void put(std::vector<uint8_t>& v, T x) {
    uint8_t b[sizeof(T)];
    memcpy(b, &x, sizeof(T));  // little-endian host (x86-64 / aarch64)
    v.insert(v.end(), b, b + sizeof(T));
}

// SAM spec 5.3: the UCSC binning scheme
int reg2bin(int64_t beg, int64_t end) {
    --end;
    if (beg >> 14 == end >> 14) return (int)(((1 << 15) - 1) / 7 + (beg >> 14));
    if (beg >> 17 == end >> 17) return (int)(((1 << 12) - 1) / 7 + (beg >> 17));
    if (beg >> 20 == end >> 20) return (int)(((1 << 9) - 1) / 7 + (beg >> 20));
    if (beg >> 23 == end >> 23) return (int)(((1 << 6) - 1) / 7 + (beg >> 23));
    if (beg >> 26 == end >> 26) return (int)(((1 << 3) - 1) / 7 + (beg >> 26));
    return 0;
}

int aux_type_size(char x) {  // sam_utils.h:24-30
    if (x == 'C' || x == 'c' || x == 'A') return 1;
    if (x == 'S' || x == 's') return 2;
    if (x == 'I' || x == 'i' || x == 'f') return 4;
    if (x == 'd') return 8;
    return 0;
}

}  // namespace

// ---- raw byte source ----------------------------------------------------------------------------------------------------
// plain text / gzip: zlib's gz* layer.  BGZF (every BAM, bgzip'ed SAM): the file is a sequence of independent deflate blocks
// of <= 64 KB, so a producer thread reads the compressed blocks in order and inflates a batch of them on g_io_threads
// worker threads straight into the batch's final buffer (offsets = prefix sums of the blocks' ISIZE fields) while the
// consumer parses the previous batch.  The reference reads its input with htslib's single-threaded BGZF reader.
struct AlnReader::Source {
    gzFile gz = nullptr;
    std::vector<uint8_t> buf;
    size_t at = 0, end = 0;
    bool eof = false;

    // BGZF mode
    FILE* fp = nullptr;
    std::thread producer;
    std::mutex mu;
    std::condition_variable cv;
    std::deque<std::vector<uint8_t>> ready;   // decoded batches, in file order
    std::vector<std::vector<uint8_t>> spare;  // consumed batch buffers, handed back to the producer (no re-allocation, no page faults)
    bool done = false, stop = false;

    static bool looks_like_bgzf(const uint8_t* h, size_t n) {
        return n >= 18 && h[0] == 0x1f && h[1] == 0x8b && h[2] == 8 && (h[3] & 4) && h[12] == 'B' && h[13] == 'C' && h[14] == 2 && h[15] == 0;
    }
    void start_bgzf(const std::string& path) {
        fp = fopen(path.c_str(), "rb");
        if (!fp) die("Cannot open " + path + "! It may not exist.");
        producer = std::thread([this]() { produce(); });
    }
    // one batch: up to kBlocks compressed blocks read in order, inflated in parallel
    void produce() {
        constexpr size_t kBlocks = 512;
        struct Blk { size_t c_off, c_len, u_off, u_len; };
        std::vector<uint8_t> comp;
        std::vector<Blk> blks;
        bool file_end = false;
        while (!file_end) {
            comp.clear();
            blks.clear();
            size_t u_total = 0;
            while (blks.size() < kBlocks) {
                uint8_t h[12];
                const size_t got = fread(h, 1, 12, fp);
                if (got == 0) { file_end = true; break; }
                if (got != 12 || h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || !(h[3] & 4)) die("Corrupt BGZF block header in the alignment file!");
                const size_t xlen = rd_u16(h + 10);
                uint8_t extra[256];
                if (xlen > sizeof extra || fread(extra, 1, xlen, fp) != xlen) die("Corrupt BGZF block header in the alignment file!");
                size_t bsize = 0;
                for (size_t k = 0; k + 4 <= xlen;) {
                    const size_t slen = rd_u16(extra + k + 2);
                    if (extra[k] == 'B' && extra[k + 1] == 'C' && slen == 2) bsize = (size_t)rd_u16(extra + k + 4) + 1;
                    k += 4 + slen;
                }
                if (bsize < 12 + xlen + 8) die("Corrupt BGZF block (no BC field) in the alignment file!");
                const size_t rest = bsize - 12 - xlen;   // deflate data + CRC32 + ISIZE
                const size_t c_off = comp.size();
                comp.resize(c_off + rest);
                if (fread(comp.data() + c_off, 1, rest, fp) != rest) die("Truncated BGZF block in the alignment file!");
                const size_t u_len = rd_u32(comp.data() + c_off + rest - 4);
                if (u_len > 65536) die("Corrupt BGZF block (ISIZE) in the alignment file!");
                blks.push_back(Blk{c_off, rest - 8, u_total, u_len});
                u_total += u_len;
            }
            if (!blks.empty()) {
                std::vector<uint8_t> out;
                {
                    std::lock_guard<std::mutex> lk(mu);
                    if (!spare.empty()) { out.swap(spare.back()); spare.pop_back(); }
                }
                out.resize(u_total);
                std::atomic<size_t> next(0);
                std::atomic<int> bad(0);
                auto work = [&]() {
                    z_stream zs;
                    for (;;) {
                        const size_t i = next.fetch_add(1);
                        if (i >= blks.size()) break;
                        const Blk& k = blks[i];
                        if (k.u_len == 0) continue;
                        memset(&zs, 0, sizeof zs);
                        if (inflateInit2(&zs, -15) != Z_OK) { bad = 1; continue; }
                        zs.next_in = comp.data() + k.c_off;
                        zs.avail_in = (uInt)k.c_len;
                        zs.next_out = out.data() + k.u_off;
                        zs.avail_out = (uInt)k.u_len;
                        const int rc = inflate(&zs, Z_FINISH);
                        if (rc != Z_STREAM_END || zs.total_out != k.u_len) bad = 1;
                        inflateEnd(&zs);
                    }
                };
                const int nt = (int)std::min<size_t>((size_t)std::max(1, g_io_threads), blks.size());
                if (nt <= 1) work();
                else {
                    std::vector<std::thread> pool;
                    for (int t = 0; t < nt; ++t) pool.emplace_back(work);
                    for (auto& t : pool) t.join();
                }
                if (bad) die("Error while reading the alignment file (corrupt gzip / BGZF stream)!");
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&]() { return ready.size() < 3 || stop; });
                if (stop) return;
                ready.push_back(std::move(out));
                cv.notify_all();
            }
        }
        std::lock_guard<std::mutex> lk(mu);
        done = true;
        cv.notify_all();
    }
    ~Source() {
        if (producer.joinable()) {
            { std::lock_guard<std::mutex> lk(mu); stop = true; }
            cv.notify_all();
            producer.join();
        }
        if (fp) fclose(fp);
        if (gz) gzclose(gz);
    }

    bool fill() {
        if (eof) return false;
        if (fp) {   // BGZF: callers come here only with an empty buffer
            std::unique_lock<std::mutex> lk(mu);
            for (;;) {
                cv.wait(lk, [&]() { return !ready.empty() || done; });
                if (ready.empty()) { eof = true; return false; }
                if (buf.capacity()) { spare.emplace_back(); spare.back().swap(buf); }
                buf = std::move(ready.front());
                ready.pop_front();
                cv.notify_all();
                if (!buf.empty()) break;
            }
            at = 0;
            end = buf.size();
            return true;
        }
        if (at < end) memmove(buf.data(), buf.data() + at, end - at);
        end -= at;
        at = 0;
        const int n = gzread(gz, buf.data() + end, (unsigned)(buf.size() - end));
        if (n < 0) die("Error while reading the alignment file (corrupt gzip / BGZF stream)!");
        if (n == 0) { eof = true; return false; }
        end += (size_t)n;
        return true;
    }
    bool lenient = false;   // read() returns false, rather than stopping, when the file ends inside the n bytes
    bool read(void* dst, size_t n) {  // exactly n bytes, false at a clean EOF before the first byte
        uint8_t* d = static_cast<uint8_t*>(dst);
        size_t got = 0;
        while (got < n) {
            if (at == end && !fill()) {
                if (got == 0 || lenient) return false;
                die("Truncated BAM file!");
            }
            const size_t k = std::min(n - got, end - at);
            memcpy(d + got, buf.data() + at, k);
            at += k;
            got += k;
        }
        return true;
    }
    // one text line without the terminator: [*p, *p + *n) points into the buffer when the line lies inside it (the common
    // case), otherwise into `spill`
    bool line_view(const char*& p, size_t& n, std::string& spill) {
        if (at == end && !fill()) return false;
        const uint8_t* nl = static_cast<const uint8_t*>(memchr(buf.data() + at, '\n', end - at));
        if (nl) {
            p = reinterpret_cast<const char*>(buf.data() + at);
            n = (size_t)(nl - (buf.data() + at));
            at += n + 1;
        } else {   // the line crosses a buffer boundary
            spill.assign(reinterpret_cast<const char*>(buf.data() + at), end - at);
            at = end;
            for (;;) {
                if (at == end && !fill()) break;
                const uint8_t* q = static_cast<const uint8_t*>(memchr(buf.data() + at, '\n', end - at));
                if (q) {
                    spill.append(reinterpret_cast<const char*>(buf.data() + at), (size_t)(q - (buf.data() + at)));
                    at = (size_t)(q - buf.data()) + 1;
                    break;
                }
                spill.append(reinterpret_cast<const char*>(buf.data() + at), end - at);
                at = end;
            }
            if (spill.empty() && eof) return false;
            p = spill.data();
            n = spill.size();
        }
        if (n && p[n - 1] == '\r') --n;
        return true;
    }
    bool line(std::string& out) {
        const char* p;
        size_t n;
        std::string spill;
        if (!line_view(p, n, spill)) { out.clear(); return false; }
        out.assign(p, n);
        return true;
    }
};

// SAM text -> records on worker threads (conv_run / conv_next below)
struct AlnReader::Conv {
    std::thread th;
    std::mutex mu;
    std::condition_variable cv;
    std::deque<std::vector<uint8_t>> ready;
    std::vector<std::vector<uint8_t>> spare;
    bool done = false, stop = false;
    std::vector<uint8_t> cur;   // consumer side
    size_t at = 0;
    ~Conv() {
        if (th.joinable()) {
            { std::lock_guard<std::mutex> lk(mu); stop = true; }
            cv.notify_all();
            th.join();
        }
    }
};

AlnReader::AlnReader(const std::string& path, const char* tool, bool htslib_header) : src_(new Source) {
    FILE* probe = fopen(path.c_str(), "rb");
    if (!probe) die("Cannot open " + path + "! It may not exist.");
    uint8_t magic[4] = {0, 0, 0, 0};
    const size_t got = fread(magic, 1, 4, probe);
    fclose(probe);
    if (got >= 4 && !memcmp(magic, "CRAM", 4)) {
        if (!tool) die("rsem-run-em (H100): CRAM input for -b is not supported; convert it to BAM (convert-sam-for-rsem).");
        die(std::string(tool) + " (H100): CRAM input is not supported; convert it to BAM.");
    }
    uint8_t head[18] = {0};
    {
        FILE* p2 = fopen(path.c_str(), "rb");
        const size_t hn = p2 ? fread(head, 1, 18, p2) : 0;
        if (p2) fclose(p2);
        if (Source::looks_like_bgzf(head, hn)) src_->start_bgzf(path);
    }
    if (!src_->fp) {
        src_->gz = gzopen(path.c_str(), "rb");
        if (!src_->gz) die("Cannot open " + path + "! It may not exist.");
        gzbuffer(src_->gz, 1 << 20);
        src_->buf.resize(4 << 20);
    }
    // BAM = gzip stream whose payload starts with "BAM\1"; anything else is SAM text
    uint8_t m4[4];
    src_->fill();
    is_bam_ = src_->end - src_->at >= 4 && !memcmp(src_->buf.data() + src_->at, "BAM\1", 4);
    // a BAM header cut short
    auto truncated = [htslib_header]() {
        if (!htslib_header) die("Truncated BAM header!");
        fprintf(stderr, "[E::bam_hdr_read] truncated bam header\n");
        die("Cannot load SAM header!");
    };
    if (is_bam_) {
        src_->lenient = htslib_header;
        src_->read(m4, 4);
        uint8_t b4[4];
        if (!src_->read(b4, 4)) truncated();
        const uint32_t l_text = rd_u32(b4);
        text_.resize(l_text);
        if (l_text && !src_->read(&text_[0], l_text)) truncated();
        while (!text_.empty() && text_.back() == '\0') text_.pop_back();
        if (!src_->read(b4, 4)) truncated();
        const uint32_t n_ref = rd_u32(b4);
        for (uint32_t i = 0; i < n_ref; ++i) {
            if (!src_->read(b4, 4)) truncated();
            const uint32_t l_name = rd_u32(b4);
            std::string name(l_name, '\0');
            if (!src_->read(&name[0], l_name)) truncated();
            while (!name.empty() && name.back() == '\0') name.pop_back();
            if (!src_->read(b4, 4)) truncated();
            ref_names_.push_back(name);
            ref_lens_.push_back(rd_u32(b4));
        }
        src_->lenient = false;
    } else {
        // header lines up to the first alignment line (kept as the pending line)
        std::string ln;
        while (src_->line(ln)) {
            if (ln.empty()) continue;
            if (ln[0] != '@') { pending_ = ln; have_pending_ = true; break; }
            text_ += ln;
            text_ += '\n';
            if (ln.compare(0, 3, "@SQ") == 0) {
                std::string name;
                uint32_t len = 0;
                size_t fr = 4;
                while (fr < ln.size()) {
                    size_t to = ln.find('\t', fr);
                    if (to == std::string::npos) to = ln.size();
                    if (ln.compare(fr, 3, "SN:") == 0) name = ln.substr(fr + 3, to - fr - 3);
                    else if (ln.compare(fr, 3, "LN:") == 0) len = (uint32_t)strtoul(ln.c_str() + fr + 3, nullptr, 10);
                    fr = to + 1;
                }
                ref_names_.push_back(name);
                ref_lens_.push_back(len);
            }
        }
    }
    for (size_t i = 0; i < ref_names_.size(); ++i) ref_index_[ref_names_[i]] = (int)i;
    if (!is_bam_) {
        conv_ = new Conv;
        conv_->th = std::thread([this]() { conv_run(); });
    }
}

AlnReader::~AlnReader() {
    delete conv_;   // joins the converter, which uses src_
    delete src_;
}

bool AlnReader::next(BamRecord& rec) {
    if (is_bam_) {
        uint8_t b4[4];
        if (!src_->read(b4, 4)) return false;
        const uint32_t block = rd_u32(b4);
        if (block < 32) die("Corrupt BAM record!");
        rec.data.resize(block);
        if (!src_->read(rec.data.data(), block)) die("Truncated BAM file!");
        return true;
    }
    return conv_next(rec);
}

// ---- SAM text -> records, pipelined -------------------------------------------------------------------------------------
// A converter thread takes the text behind the header in chunks of ~16 MB that end at a line boundary, has g_io_threads
// workers turn the lines of a chunk into BAM-encoded records (u32 size + bytes, the BAM stream format) in parallel and queues
// the result in file order; next() only frames records out of those buffers.  The reference parses SAM text on one thread.
void AlnReader::conv_run() {
    Conv& c = *conv_;
    constexpr size_t kChunk = 16u << 20;
    std::string text;
    if (have_pending_) { text = pending_; text += '\n'; have_pending_ = false; }
    bool input_end = false;
    std::vector<std::vector<uint8_t>> part;
    while (!input_end || !text.empty()) {
        // fill up to kChunk from the source (this thread is the only user of src_ from here on)
        while (!input_end && text.size() < kChunk) {
            if (src_->at == src_->end && !src_->fill()) { input_end = true; break; }
            text.append(reinterpret_cast<const char*>(src_->buf.data() + src_->at), src_->end - src_->at);
            src_->at = src_->end;
        }
        size_t use = text.size();
        if (!input_end) {
            const size_t nl = text.rfind('\n');
            if (nl == std::string::npos) continue;   // a single line longer than the chunk: keep reading
            use = nl + 1;
        }
        if (use == 0) break;
        // line-aligned ranges for the workers
        const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, g_io_threads), use / (256u << 10) + 1));
        std::vector<size_t> cut((size_t)T + 1, use);
        cut[0] = 0;
        for (int t = 1; t < T; ++t) {
            size_t p = use * (size_t)t / (size_t)T;
            const size_t nl = text.find('\n', p);
            cut[(size_t)t] = (nl == std::string::npos || nl + 1 > use) ? use : nl + 1;
        }
        part.resize((size_t)T);
        auto work = [&](int t) {
            std::vector<uint8_t>& out = part[(size_t)t];
            out.clear();
            BamRecord rec;
            int last_ref = -1;
            const char* p = text.data() + cut[(size_t)t];
            const char* e = text.data() + cut[(size_t)t + 1];
            while (p < e) {
                const char* nl = static_cast<const char*>(memchr(p, '\n', (size_t)(e - p)));
                const char* le = nl ? nl : e;
                size_t n = (size_t)(le - p);
                if (n && p[n - 1] == '\r') --n;
                if (n) {
                    parse_sam_line(p, n, rec, last_ref);
                    const uint32_t sz = (uint32_t)rec.data.size();
                    const size_t at = out.size();
                    out.resize(at + 4 + sz);
                    wr_u32(out.data() + at, sz);
                    memcpy(out.data() + at + 4, rec.data.data(), sz);
                }
                p = nl ? nl + 1 : e;
            }
        };
        if (T == 1) work(0);
        else {
            std::vector<std::thread> pool;
            for (int t = 0; t < T; ++t) pool.emplace_back(work, t);
            for (auto& th : pool) th.join();
        }
        size_t total = 0;
        for (int t = 0; t < T; ++t) total += part[(size_t)t].size();
        std::vector<uint8_t> out;
        {
            std::lock_guard<std::mutex> lk(c.mu);
            if (!c.spare.empty()) { out.swap(c.spare.back()); c.spare.pop_back(); }
        }
        out.resize(total);
        size_t at = 0;
        for (int t = 0; t < T; ++t) {
            if (!part[(size_t)t].empty()) memcpy(out.data() + at, part[(size_t)t].data(), part[(size_t)t].size());
            at += part[(size_t)t].size();
        }
        text.erase(0, use);
        if (total) {
            std::unique_lock<std::mutex> lk(c.mu);
            c.cv.wait(lk, [&]() { return c.ready.size() < 3 || c.stop; });
            if (c.stop) return;
            c.ready.push_back(std::move(out));
            c.cv.notify_all();
        }
    }
    std::lock_guard<std::mutex> lk(c.mu);
    c.done = true;
    c.cv.notify_all();
}

bool AlnReader::conv_next(BamRecord& rec) {
    Conv& c = *conv_;
    if (c.at == c.cur.size()) {
        std::unique_lock<std::mutex> lk(c.mu);
        c.cv.wait(lk, [&]() { return !c.ready.empty() || c.done; });
        if (c.ready.empty()) return false;
        if (c.cur.capacity()) { c.spare.emplace_back(); c.spare.back().swap(c.cur); }
        c.cur = std::move(c.ready.front());
        c.ready.pop_front();
        c.at = 0;
        c.cv.notify_all();
    }
    const uint32_t sz = rd_u32(c.cur.data() + c.at);
    rec.data.assign(c.cur.data() + c.at + 4, c.cur.data() + c.at + 4 + sz);
    c.at += 4 + (size_t)sz;
    return true;
}

// SAM text -> BAM record (SAM spec section 4.2; field encodings as htslib's sam_parse1 chooses them).  No allocation per
// line: fields are (pointer, length) views into the reader's buffer, the record's byte vector is reused by the caller.
void AlnReader::parse_sam_line(const char* ln, size_t len, BamRecord& rec, int& last_ref_) const {
    struct Fld { const char* p; size_t n; };
    Fld f[11];
    const char* end = ln + len;
    const char* q = ln;
    int nf = 0;
    while (nf < 11) {
        const char* t = static_cast<const char*>(memchr(q, '\t', (size_t)(end - q)));
        f[nf].p = q;
        f[nf].n = (size_t)((t ? t : end) - q);
        ++nf;
        if (!t) { q = end; break; }
        q = t + 1;
    }
    if (nf < 11) die("Malformed SAM line (fewer than 11 fields): " + std::string(ln, std::min<size_t>(len, 80)));
    const char* opt = (f[10].p + f[10].n < end) ? f[10].p + f[10].n + 1 : end;   // first optional field
    auto to_i64 = [](const Fld& x) {   // atoll on a view
        const char* s = x.p;
        const char* e = x.p + x.n;
        bool neg = false;
        if (s < e && (*s == '-' || *s == '+')) { neg = *s == '-'; ++s; }
        long long v = 0;
        while (s < e && *s >= '0' && *s <= '9') v = v * 10 + (*s++ - '0');
        return neg ? -v : v;
    };
    auto is = [](const Fld& x, char c) { return x.n == 1 && x.p[0] == c; };
    const Fld &qname = f[0], &rname = f[2], &cigar = f[5], &rnext = f[6], &seq = f[9], &qual = f[10];
    const int flag = (int)to_i64(f[1]);
    const int64_t pos = to_i64(f[3]) - 1, pnext = to_i64(f[7]) - 1, tlen = to_i64(f[8]);
    const int mapq = (int)to_i64(f[4]);
    auto ref_id = [&](const Fld& x) -> int {
        if (is(x, '*')) return -1;
        if (last_ref_ >= 0 && ref_names_[(size_t)last_ref_].size() == x.n && !memcmp(ref_names_[(size_t)last_ref_].data(), x.p, x.n))
            return last_ref_;
        auto it = ref_index_.find(std::string(x.p, x.n));
        if (it == ref_index_.end()) die("SAM line refers to a reference sequence that is not in the header: " + std::string(x.p, x.n));
        last_ref_ = it->second;
        return it->second;
    };
    const int tid = ref_id(rname);
    const int mtid = is(rnext, '=') ? tid : ref_id(rnext);
    // CIGAR
    uint32_t cig[64];
    std::vector<uint32_t> cig_big;
    size_t n_cig = 0;
    int64_t ref_len = 0;
    if (!is(cigar, '*')) {
        const char* p = cigar.p;
        const char* e = cigar.p + cigar.n;
        while (p < e) {
            unsigned long n = 0;
            const char* d0 = p;
            while (p < e && *p >= '0' && *p <= '9') n = n * 10 + (unsigned long)(*p++ - '0');
            uint32_t op;
            switch (p < e ? *p : 0) {
                case 'M': op = 0; break; case 'I': op = 1; break; case 'D': op = 2; break; case 'N': op = 3; break;
                case 'S': op = 4; break; case 'H': op = 5; break; case 'P': op = 6; break; case '=': op = 7; break;
                case 'X': op = 8; break;
                default: op = 99;
            }
            if (p == d0 || op == 99) die("Malformed CIGAR string: " + std::string(cigar.p, cigar.n));
            const uint32_t w = (uint32_t)(n << 4) | op;
            if (n_cig < 64) cig[n_cig] = w;
            else { if (n_cig == 64) cig_big.assign(cig, cig + 64); cig_big.push_back(w); }
            ++n_cig;
            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) ref_len += (int64_t)n;
            ++p;
        }
    }
    const uint32_t* cg = n_cig > 64 ? cig_big.data() : cig;
    const int l_seq = is(seq, '*') ? 0 : (int)seq.n;
    std::vector<uint8_t>& d = rec.data;
    const size_t fixed = 32 + qname.n + 1 + n_cig * 4 + ((size_t)l_seq + 1) / 2 + (size_t)l_seq;
    d.resize(fixed);
    uint8_t* w = d.data();
    const int64_t endp = (flag & 4) || n_cig == 0 || ref_len == 0 ? pos + 1 : pos + ref_len;
    wr_u32(w, (uint32_t)tid);
    wr_u32(w + 4, (uint32_t)(int32_t)pos);
    // an unplaced record (pos = -1) gets bin 4680 = reg2bin(-1, 0), as htslib computes it
    wr_u32(w + 8, ((uint32_t)reg2bin(pos, endp) << 16) | ((uint32_t)(mapq & 255) << 8) | (uint32_t)(qname.n + 1));
    wr_u32(w + 12, ((uint32_t)flag << 16) | (uint32_t)n_cig);
    wr_u32(w + 16, (uint32_t)l_seq);
    wr_u32(w + 20, (uint32_t)mtid);
    wr_u32(w + 24, (uint32_t)(int32_t)pnext);
    wr_u32(w + 28, (uint32_t)(int32_t)tlen);
    w += 32;
    memcpy(w, qname.p, qname.n);
    w += qname.n;
    *w++ = 0;
    for (size_t i = 0; i < n_cig; ++i) { wr_u32(w, cg[i]); w += 4; }
    struct Nt16 {   // letter -> 4-bit code; built once (thread-safe static initialisation: worker threads call this function)
        uint8_t v[256];
        Nt16() {
            memset(v, 15, sizeof v);
            const char* code = "=ACMGRSVTWYHKDBN";
            for (int i = 0; i < 16; ++i) { v[(uint8_t)code[i]] = (uint8_t)i; v[(uint8_t)tolower(code[i])] = (uint8_t)i; }
        }
    };
    static const Nt16 nt16_table;
    const uint8_t* nt16 = nt16_table.v;
    for (int i = 0; i < l_seq; i += 2) {
        const uint8_t hi = nt16[(uint8_t)seq.p[i]], lo = i + 1 < l_seq ? nt16[(uint8_t)seq.p[i + 1]] : 0;
        *w++ = (uint8_t)(hi << 4 | lo);
    }
    if (is(qual, '*')) { memset(w, 0xff, (size_t)l_seq); w += l_seq; }
    else {
        if ((int)qual.n != l_seq) die("SAM line with SEQ and QUAL of different lengths: " + std::string(qname.p, qname.n));
        for (int i = 0; i < l_seq; ++i) *w++ = (uint8_t)(qual.p[i] - 33);
    }
    // optional fields
    for (const char* a = opt; a < end;) {
        const char* t = static_cast<const char*>(memchr(a, '\t', (size_t)(end - a)));
        const char* b = t ? t : end;
        if (b - a < 5 || a[2] != ':' || a[4] != ':') die("Malformed optional SAM field in the line of " + std::string(qname.p, qname.n));
        const char type = a[3];
        const std::string val(a + 5, (size_t)(b - a - 5));
        d.push_back((uint8_t)a[0]);
        d.push_back((uint8_t)a[1]);
        if (type == 'A') { d.push_back('A'); d.push_back((uint8_t)(val.empty() ? ' ' : val[0])); }
        else if (type == 'i') {
            const long long x = atoll(val.c_str());
            if (x < 0) {
                if (x >= -128) { d.push_back('c'); put<int8_t>(d, (int8_t)x); }
                else if (x >= -32768) { d.push_back('s'); put<int16_t>(d, (int16_t)x); }
                else { d.push_back('i'); put<int32_t>(d, (int32_t)x); }
            } else {
                if (x <= 255) { d.push_back('C'); put<uint8_t>(d, (uint8_t)x); }
                else if (x <= 65535) { d.push_back('S'); put<uint16_t>(d, (uint16_t)x); }
                else { d.push_back('I'); put<uint32_t>(d, (uint32_t)x); }
            }
        } else if (type == 'f') { d.push_back('f'); put<float>(d, (float)atof(val.c_str())); }
        else if (type == 'd') { d.push_back('d'); put<double>(d, atof(val.c_str())); }
        else if (type == 'Z' || type == 'H') {
            d.push_back((uint8_t)type);
            d.insert(d.end(), val.begin(), val.end());
            d.push_back(0);
        } else if (type == 'B') {
            if (val.empty()) die("Malformed B-type optional field in the line of " + std::string(qname.p, qname.n));
            const char sub = val[0];
            std::vector<std::string> items;
            for (size_t fr = 1; fr < val.size();) {
                if (val[fr] == ',') ++fr;
                size_t to = val.find(',', fr);
                if (to == std::string::npos) to = val.size();
                if (to > fr) items.push_back(val.substr(fr, to - fr));
                fr = to;
            }
            d.push_back('B');
            d.push_back((uint8_t)sub);
            put<uint32_t>(d, (uint32_t)items.size());
            for (const std::string& it : items) {
                switch (sub) {
                    case 'c': put<int8_t>(d, (int8_t)atoi(it.c_str())); break;
                    case 'C': put<uint8_t>(d, (uint8_t)atoi(it.c_str())); break;
                    case 's': put<int16_t>(d, (int16_t)atoi(it.c_str())); break;
                    case 'S': put<uint16_t>(d, (uint16_t)atoi(it.c_str())); break;
                    case 'i': put<int32_t>(d, (int32_t)atoll(it.c_str())); break;
                    case 'I': put<uint32_t>(d, (uint32_t)atoll(it.c_str())); break;
                    case 'f': put<float>(d, (float)atof(it.c_str())); break;
                    default: die("Unknown B-array subtype in the line of " + std::string(qname.p, qname.n));
                }
            }
        } else die("Unknown optional field type in the line of " + std::string(qname.p, qname.n));
        a = t ? t + 1 : end;
    }
}

// ---- BamRecord helpers ------------------------------------------------------------------------------------------------
uint16_t BamRecord::flag() const { return (uint16_t)(rd_u32(data.data() + 12) >> 16); }
int32_t BamRecord::tid() const { return (int32_t)rd_u32(data.data()); }
int32_t BamRecord::pos() const { return (int32_t)rd_u32(data.data() + 4); }
int32_t BamRecord::l_seq() const { return (int32_t)rd_u32(data.data() + 16); }
const char* BamRecord::qname() const { return reinterpret_cast<const char*>(data.data() + 32); }
uint32_t BamRecord::n_cigar() const { return rd_u32(data.data() + 12) & 0xffff; }
uint32_t BamRecord::cigar(uint32_t i) const { return rd_u32(data.data() + 32 + data[8] + 4 * (size_t)i); }
int BamRecord::base4(int32_t i) const {
    const uint8_t b = data[32 + data[8] + 4 * (size_t)n_cigar() + (size_t)(i >> 1)];
    return (i & 1) ? (b & 15) : (b >> 4);
}
const uint8_t* BamRecord::qual() const { return data.data() + 32 + data[8] + 4 * (size_t)n_cigar() + ((size_t)l_seq() + 1) / 2; }

// bam_aux_get + bam_aux2i of htslib 1.3 (SamParser.h:63-68 reads the aligner's "too many alignments" tag with them):
// the first field with this tag; its value if the type is one of cCsSiI, 0 for any other type
bool BamRecord::aux_int(const char tag[2], long long& value) const {
    size_t at = 32 + data[8] + 4 * (size_t)n_cigar() + ((size_t)l_seq() + 1) / 2 + (size_t)l_seq();
    while (at + 3 <= data.size()) {
        const char t0 = (char)data[at], t1 = (char)data[at + 1], type = (char)data[at + 2];
        const size_t val_at = at + 3;
        size_t len;
        if (type == 'Z' || type == 'H') {
            len = 0;
            while (val_at + len < data.size() && data[val_at + len]) ++len;
            ++len;
        } else if (type == 'B') {
            if (val_at + 5 > data.size()) die("Corrupt optional field in a BAM record!");
            len = 5 + (size_t)aux_type_size((char)data[val_at]) * rd_u32(data.data() + val_at + 1);
        } else {
            len = (size_t)aux_type_size(type);
            if (len == 0) die("Corrupt optional field in a BAM record!");
        }
        if (val_at + len > data.size()) die("Corrupt optional field in a BAM record!");
        if (t0 == tag[0] && t1 == tag[1]) {
            const uint8_t* v = data.data() + val_at;
            switch (type) {
                case 'c': value = (int8_t)v[0]; break;
                case 'C': value = v[0]; break;
                case 's': value = (int16_t)rd_u16(v); break;
                case 'S': value = rd_u16(v); break;
                case 'i': value = (int32_t)rd_u32(v); break;
                case 'I': value = rd_u32(v); break;
                default: value = 0;
            }
            return true;
        }
        at = val_at + len;
    }
    return false;
}

// MAPQ + ZW:f from the posterior (BamWriter.h:39-48, sam_utils.h:72-76)
uint8_t prb_to_mapq(double prb) {
    const double err = 1.0 - prb;
    return err <= 1e-10 ? 100 : (uint8_t)(-10 * std::log10(err) + .5);
}

std::vector<float> mapq_thresholds() {
    std::vector<float> t(101, 0.0f);
    const uint32_t hi = 0x40000000u;   // 2.0f; every p >= 1 gives 100
    for (int m = 1; m <= 100; ++m) {   // bisection over the ordered bit patterns of the non-negative floats
        uint32_t lo = 0, up = hi;
        while (lo < up) {
            const uint32_t mid = lo + (up - lo) / 2;
            float p;
            memcpy(&p, &mid, 4);
            if (prb_to_mapq(p) >= m) up = mid;
            else lo = mid + 1;
        }
        memcpy(&t[m], &lo, 4);
    }
    return t;
}

void BamRecord::set_alignment_weight(double prb) {
    data[9] = prb_to_mapq(prb);  // bin_mq_nl: byte 8 = l_read_name, byte 9 = MAPQ
    const float val = (float)prb;
    // walk the optional fields to find an existing ZW
    const uint32_t l_name = data[8], n_cig = rd_u32(data.data() + 12) & 0xffff;
    const int32_t l_seq = (int32_t)rd_u32(data.data() + 16);
    size_t at = 32 + l_name + 4 * (size_t)n_cig + ((size_t)l_seq + 1) / 2 + (size_t)l_seq;
    while (at + 3 <= data.size()) {
        const char t0 = (char)data[at], t1 = (char)data[at + 1], type = (char)data[at + 2];
        size_t val_at = at + 3, len;
        if (type == 'Z' || type == 'H') {
            len = 0;
            while (val_at + len < data.size() && data[val_at + len]) ++len;
            ++len;
        } else if (type == 'B') {
            const int sz = aux_type_size((char)data[val_at]);
            len = 5 + (size_t)sz * rd_u32(data.data() + val_at + 1);
        } else {
            len = (size_t)aux_type_size(type);
            if (len == 0) die("Corrupt optional field in a BAM record!");
        }
        if (t0 == 'Z' && t1 == 'W') {
            memcpy(&data[val_at], &val, 4);  // the reference overwrites 4 bytes whatever the stored type is
            return;
        }
        at = val_at + len;
    }
    data.push_back('Z');
    data.push_back('W');
    data.push_back('f');
    put<float>(data, val);
}

// ---- header text as the reference rewrites it (SamHeader.cpp:74-114 + insertPG, SamHeader.hpp:38-60) -------------------
std::string rsem_bam_header_text(const std::string& in_text, const std::string& pg_id, const std::string& pg_cl,
                                 const std::string* sq, bool reference_pg_ids) {
    std::string HD, SQ, RG, PG, CO, other;
    std::vector<std::string> pids;
    size_t fr = 0;
    while (fr < in_text.size()) {
        size_t to = in_text.find('\n', fr);
        if (to == std::string::npos) to = in_text.size();
        const std::string line = in_text.substr(fr, to - fr);
        fr = to + 1;
        if (line.empty() || line[0] != '@') continue;
        const std::string tag = line.substr(1, 2);
        if (tag == "HD") {
            if (!HD.empty()) die("@HD tag can only present once!");
            HD = line + "\n";
        } else if (tag == "SQ") SQ += line + "\n";
        else if (tag == "RG") RG += line + "\n";
        else if (tag == "PG") {
            std::string id;
            bool has_id = false;
            for (size_t a = 4; a < line.size();) {
                size_t b = line.find('\t', a);
                if (line.compare(a, 3, "ID:") == 0) {
                    // SamHeader::parse_line takes line.substr(fr, to) with `to` an index
                    id = reference_pg_ids ? line.substr(a, b).substr(3) : line.substr(a + 3, (b == std::string::npos ? line.size() : b) - a - 3);
                    has_id = true;
                }
                if (b == std::string::npos) break;
                a = b + 1;
            }
            if (reference_pg_ids && !has_id) die("\"" + line + "\" does not contain an ID!");
            if (std::find(pids.begin(), pids.end(), id) != pids.end()) die("Program record identifier " + id + " is not unique!");
            pids.push_back(id);
            PG += line + "\n";
        } else if (tag == "CO") CO += line + "\n";
        else other += line;  // sic: the reference appends these lines without their newline (SamHeader.cpp:111)
    }
    if (sq) SQ = *sq;
    if (std::find(pids.begin(), pids.end(), pg_id) == pids.end()) PG += "@PG\tID:" + pg_id + (pg_cl.empty() ? "" : "\tCL:" + pg_cl) + "\n";
    return HD + SQ + RG + PG + CO + other;
}

// ---- BGZF writer ----------------------------------------------------------------------------------------------------------
namespace {
constexpr size_t kBgzfBlock = 0xff00;

void bgzf_compress(const uint8_t* src, size_t n, std::vector<uint8_t>& out) {
    out.resize(18 + compressBound((uLong)n) + 8);
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (deflateInit2(&zs, Z_DEFAULT_COMPRESSION, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) die("zlib: deflateInit2 failed");
    zs.next_in = const_cast<Bytef*>(src);
    zs.avail_in = (uInt)n;
    zs.next_out = out.data() + 18;
    zs.avail_out = (uInt)(out.size() - 18 - 8);
    if (deflate(&zs, Z_FINISH) != Z_STREAM_END) die("zlib: deflate failed");
    const size_t clen = zs.total_out;
    deflateEnd(&zs);
    static const uint8_t hdr[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
    memcpy(out.data(), hdr, 16);
    wr_u16(out.data() + 16, (uint16_t)(18 + clen + 8 - 1));
    wr_u32(out.data() + 18 + clen, (uint32_t)crc32(crc32(0L, Z_NULL, 0), src, (uInt)n));
    wr_u32(out.data() + 18 + clen + 4, (uint32_t)n);
    out.resize(18 + clen + 8);
}
}  // namespace

BamWriter::BamWriter(const std::string& path, const std::string& header_text, int threads) : threads_(std::max(1, threads)) {
    fo_ = fopen(path.c_str(), "wb");
    if (!fo_) die("Cannot open " + path + " for writing!");
    // references come from the @SQ lines of the (rewritten) text, like sam_hdr_parse does for the reference
    std::vector<std::pair<std::string, uint32_t>> refs;
    size_t fr = 0;
    while (fr < header_text.size()) {
        size_t to = header_text.find('\n', fr);
        if (to == std::string::npos) to = header_text.size();
        if (header_text.compare(fr, 3, "@SQ") == 0) {
            std::string name;
            uint32_t len = 0;
            for (size_t a = fr + 4; a < to;) {
                size_t b = header_text.find('\t', a);
                if (b == std::string::npos || b > to) b = to;
                if (header_text.compare(a, 3, "SN:") == 0) name = header_text.substr(a + 3, b - a - 3);
                else if (header_text.compare(a, 3, "LN:") == 0) len = (uint32_t)strtoul(header_text.c_str() + a + 3, nullptr, 10);
                a = b + 1;
            }
            refs.emplace_back(name, len);
        }
        fr = to + 1;
    }
    std::vector<uint8_t> h;
    h.insert(h.end(), {'B', 'A', 'M', 1});
    put<uint32_t>(h, (uint32_t)header_text.size());
    h.insert(h.end(), header_text.begin(), header_text.end());
    put<uint32_t>(h, (uint32_t)refs.size());
    for (auto& r : refs) {
        put<uint32_t>(h, (uint32_t)r.first.size() + 1);
        h.insert(h.end(), r.first.begin(), r.first.end());
        h.push_back(0);
        put<uint32_t>(h, r.second);
    }
    append(h.data(), h.size());
    flush_pending(true);  // htslib also ends the header in its own block
}

void BamWriter::append(const uint8_t* p, size_t n) {
    pending_.insert(pending_.end(), p, p + n);
    if (pending_.size() >= kBgzfBlock * 64 * (size_t)threads_) flush_pending(false);
}

void BamWriter::write_encoded(const uint8_t* p, size_t n) { append(p, n); }

void BamWriter::write(const BamRecord& rec) {
    uint8_t b4[4];
    wr_u32(b4, (uint32_t)rec.data.size());
    append(b4, 4);
    append(rec.data.data(), rec.data.size());
}

// compress the pending bytes block by block on the worker threads, write the blocks in order
void BamWriter::flush_pending(bool all) {
    const size_t n_blocks = all ? (pending_.size() + kBgzfBlock - 1) / kBgzfBlock : pending_.size() / kBgzfBlock;
    if (n_blocks == 0) return;
    std::vector<std::vector<uint8_t>> out(n_blocks);
    std::atomic<size_t> next(0);
    auto work = [&]() {
        for (;;) {
            const size_t i = next.fetch_add(1);
            if (i >= n_blocks) break;
            const size_t a = i * kBgzfBlock, b = std::min(pending_.size(), a + kBgzfBlock);
            bgzf_compress(pending_.data() + a, b - a, out[i]);
        }
    };
    const int nt = (int)std::min<size_t>((size_t)threads_, n_blocks);
    if (nt <= 1) work();
    else {
        std::vector<std::thread> pool;
        for (int t = 0; t < nt; ++t) pool.emplace_back(work);
        for (auto& t : pool) t.join();
    }
    for (auto& o : out)
        if (fwrite(o.data(), 1, o.size(), fo_) != o.size()) die("Error while writing the BAM file!");
    const size_t used = std::min(pending_.size(), n_blocks * kBgzfBlock);
    pending_.erase(pending_.begin(), pending_.begin() + (long)used);
}

void BamWriter::close() {
    if (!fo_) return;
    flush_pending(true);
    static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (fwrite(eof, 1, 28, fo_) != 28) die("Error while writing the BAM file!");
    if (fclose(fo_) != 0) die("Error while closing the BAM file!");
    fo_ = nullptr;
}

BamWriter::~BamWriter() { close(); }

}  // namespace host
