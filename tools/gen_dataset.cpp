// Synthetic RSEM intermediate-file generator (tooling; not part of the product path).
//
// Writes, for one sample, exactly the files `rsem-run-em` / `rsem-run-gibbs` read
// (SURVEY.md section 8(c), formats from the reference):
//   ref/r.seq   RefSeq::write layout           (/root/reference/RefSeq.h:130-138)
//   ref/r.ti    Transcripts::writeTo layout    (/root/reference/Transcripts.h:96-103, Transcript.h:148-167)
//   ref/r.grp   gene start ids                 (/root/reference/GroupInfo.h:34-53)
//   s.stat/s.cnt        "N0 N1 N2 N_tot"       (/root/reference/EM.cpp:607-613)
//   s.temp/s.mparams    ten numbers            (/root/reference/rsem-calculate-expression:606-615)
//   s.temp/s.dat        CSR text               (/root/reference/HitContainer.h:81-91, parseIt.cpp:197-211)
//   s.temp/s_alignable*.f[aq], s_un*.f[aq]     (/root/reference/utils.h:129-149)
//   s.temp/s.omit       (empty or ids)         (/root/reference/Transcripts.h:135-142)
//
// Data model: isoform families (= genes, contiguous transcript ids).  A member transcript is
// <unique prefix><shared body>, so a fragment drawn from the body aligns to every member of
// the family (real multi-mapping); fragments drawn from a prefix are unique.  Family expression
// weights are u^4 (long tailed).  Reverse-strand hits carry a negative sid and `pos` in
// reverse-strand coordinates (/root/reference/SamParser.h:136-141).
//
// Build: g++ -O2 -std=c++17 -o tools/gen_dataset tools/gen_dataset.cpp
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <sys/stat.h>
#include <vector>

namespace {

struct Rng {  // splitmix64 / xorshift-style; deterministic everywhere
    uint64_t s;
    explicit Rng(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ull + 0x1234567ull) {}
    uint64_t next() {
        uint64_t z = (s += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    }
    double uni() { return (next() >> 11) * (1.0 / 9007199254740992.0); }
    int below(int n) { return (int)(uni() * n); }
    int range(int lo, int hi) { return lo + below(hi - lo + 1); }  // inclusive
    int poisson(double lam) {
        double L = std::exp(-lam), p = 1.0;
        int k = 0;
        do { ++k; p *= uni(); } while (p > L);
        return k - 1;
    }
};

struct Cfg {
    std::string out = "dataset";
    int read_type = 0;
    int M = 200;
    long N1 = 2000, N0 = 100;
    double avg_family = 5.0;
    int read_len = 50;
    int var_len = 0;          // read lengths uniform in [read_len - var_len, read_len]
    uint64_t seed = 11;
    double probF = 0.5;
    int est_rspd = 0, B = 20;
    int polyA = 0;            // polyA tail length appended to every transcript (0 = none)
    int zipf = 0;             // family sizes ~ Zipf(1.1) truncated at 200 (config C5)
    double spurious = 0.0;    // fraction of reads given one extra random (mismatching) hit
    int frag_min = 150, frag_max = 300;
    int minL = 1, maxL = 1000;  // .mparams fragment-length bounds
    int seed_len = 25;
    double frag_mean = -1, frag_sd = 0;
    int omit = 0;             // number of trailing transcripts listed in .omit (never hit)
    double nfrac = 0.002;     // probability of an 'N' base call
    int sam = 0;              // also write <out>/aln.sam: the same reads and alignments as a SAM file the unmodified
                              // rsem-parse-alignments accepts (SamParser.h:122-265), for runs through rsem-calculate-expression
    int genome = 0;           // place every family on a chromosome as a gene locus: r.ti of type 0 with exon structures,
                              // and r.chrlist (rsem-tbam2gbam input).  Drawn from its own generator: the rest is unchanged
    int has_sample_seed = 0;  // --sample-seed: the generator is reseeded after the reference and .omit are written, so
    uint64_t sample_seed = 0; // samples share byte-identical ref/r.* and differ in expression and reads
    double expressed_frac = 1.0;  // fraction of families with non-zero expression (single-cell-like samples)
};

const char BASES[5] = {'A', 'C', 'G', 'T', 'N'};
inline char comp(char c) {
    switch (c) { case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A'; }
    return 'N';
}
std::string revcomp(const std::string& s) {
    std::string r(s.size(), 'N');
    for (size_t i = 0; i < s.size(); ++i) r[i] = comp(s[s.size() - 1 - i]);
    return r;
}
std::string randseq(Rng& g, int n) {
    std::string s(n, 'A');
    for (int i = 0; i < n; ++i) s[i] = BASES[g.below(4)];
    return s;
}

const int QVALS[5] = {20, 30, 35, 38, 40};

// sequencing: copy `tmpl`, draw qualities, introduce errors at 10^(-q/10)
void sequence(Rng& g, const std::string& tmpl, double nfrac, std::string& seq, std::string& qual) {
    seq = tmpl;
    qual.assign(tmpl.size(), 'I');
    for (size_t i = 0; i < tmpl.size(); ++i) {
        int q = QVALS[g.below(5)];
        qual[i] = (char)(33 + q);
        double pe = std::pow(10.0, -q / 10.0);
        double u = g.uni();
        if (u < nfrac) seq[i] = 'N';
        else if (u < nfrac + pe) {
            char c;
            do { c = BASES[g.below(4)]; } while (c == tmpl[i]);
            seq[i] = c;
        }
    }
}

struct Hit { int sid, pos, insertL, fwd; };  // fwd: forward-strand start of the fragment on the transcript

void die(const char* msg) { fprintf(stderr, "gen_dataset: %s\n", msg); exit(2); }
FILE* xopen(const std::string& p) {
    FILE* f = fopen(p.c_str(), "w");
    if (!f) { fprintf(stderr, "gen_dataset: cannot open %s\n", p.c_str()); exit(2); }
    static char* bufs[64]; static int nb = 0;
    if (nb < 64) { bufs[nb] = (char*)malloc(1 << 20); setvbuf(f, bufs[nb++], _IOFBF, 1 << 20); }
    return f;
}

}  // namespace

int main(int argc, char** argv) {
    Cfg c;
    for (int i = 1; i + 1 < argc; i += 2) {
        std::string k = argv[i];
        const char* v = argv[i + 1];
        if (k == "--out") c.out = v;
        else if (k == "--read-type") c.read_type = atoi(v);
        else if (k == "--M") c.M = atoi(v);
        else if (k == "--N1") c.N1 = atol(v);
        else if (k == "--N0") c.N0 = atol(v);
        else if (k == "--avg-family") c.avg_family = atof(v);
        else if (k == "--read-len") c.read_len = atoi(v);
        else if (k == "--var-len") c.var_len = atoi(v);
        else if (k == "--seed") c.seed = strtoull(v, nullptr, 10);
        else if (k == "--probF") c.probF = atof(v);
        else if (k == "--est-rspd") c.est_rspd = atoi(v);
        else if (k == "--B") c.B = atoi(v);
        else if (k == "--polyA") c.polyA = atoi(v);
        else if (k == "--zipf") c.zipf = atoi(v);
        else if (k == "--spurious") c.spurious = atof(v);
        else if (k == "--frag-min") c.frag_min = atoi(v);
        else if (k == "--frag-max") c.frag_max = atoi(v);
        else if (k == "--minL") c.minL = atoi(v);
        else if (k == "--maxL") c.maxL = atoi(v);
        else if (k == "--seed-len") c.seed_len = atoi(v);
        else if (k == "--frag-mean") c.frag_mean = atof(v);
        else if (k == "--frag-sd") c.frag_sd = atof(v);
        else if (k == "--omit") c.omit = atoi(v);
        else if (k == "--nfrac") c.nfrac = atof(v);
        else if (k == "--sam") c.sam = atoi(v);
        else if (k == "--genome") c.genome = atoi(v);
        else if (k == "--sample-seed") { c.has_sample_seed = 1; c.sample_seed = strtoull(v, nullptr, 10); }
        else if (k == "--expressed-frac") c.expressed_frac = atof(v);
        else { fprintf(stderr, "gen_dataset: unknown option %s\n", k.c_str()); return 2; }
    }
    const bool paired = c.read_type >= 2, hasQ = (c.read_type & 1);
    Rng g(c.seed);

    // ---- families / transcripts -------------------------------------------------------------
    const int Mhit = c.M - c.omit;  // transcripts that can be hit
    if (Mhit < 1) die("M - omit must be >= 1");
    std::vector<int> fam_start;     // first transcript id (1-based) of each family
    std::vector<std::string> tseq(c.M + 1);
    std::vector<int> prefix_len(c.M + 1, 0), fam_of(c.M + 1, 0);
    std::vector<std::string> body;
    {
        int t = 1;
        while (t <= c.M) {
            int sz;
            if (c.zipf) {  // Zipf(s=1.1) truncated at 200 by inversion on the discrete cdf
                static std::vector<double> cdf;
                if (cdf.empty()) { double a = 0; for (int k = 1; k <= 200; ++k) { a += std::pow(k, -1.1); cdf.push_back(a); } for (auto& x : cdf) x /= a; }
                double u = g.uni();
                sz = (int)(std::lower_bound(cdf.begin(), cdf.end(), u) - cdf.begin()) + 1;
            } else {
                sz = 1 + g.poisson(std::max(0.0, c.avg_family - 1.0));
            }
            if (t <= Mhit && t + sz - 1 > Mhit) sz = Mhit - t + 1;  // keep omitted ones in their own families
            sz = std::min(sz, c.M - t + 1);
            int need = paired ? c.frag_max + 50 : c.read_len + 50;
            int blen = std::max(need, g.range(600, 2500));
            std::string b = randseq(g, blen);
            fam_start.push_back(t);
            int f = (int)body.size();
            body.push_back(b);
            for (int k = 0; k < sz; ++k, ++t) {
                prefix_len[t] = (k == 0 && sz > 1) ? 0 : g.range(0, 300);
                if (sz == 1) prefix_len[t] = g.range(0, 300);
                tseq[t] = randseq(g, prefix_len[t]) + b;
                fam_of[t] = f;
            }
        }
        fam_start.push_back(c.M + 1);
    }
    const int F = (int)body.size();

    mkdir(c.out.c_str(), 0755);
    mkdir((c.out + "/ref").c_str(), 0755);
    mkdir((c.out + "/s.temp").c_str(), 0755);
    mkdir((c.out + "/s.stat").c_str(), 0755);

    {   // .seq  (masks: last OLEN-1 = 24 positions before the tail when polyA, RefSeq.h:31-37)
        FILE* f = xopen(c.out + "/ref/r.seq");
        for (int t = 1; t <= c.M; ++t) {
            int fullLen = (int)tseq[t].size(), totLen = fullLen + c.polyA;
            fprintf(f, "%d %d\nT%d\n%s", fullLen, totLen, t, tseq[t].c_str());
            for (int i = 0; i < c.polyA; ++i) fputc('A', f);
            fputc('\n', f);
            int nw = (fullLen - 1) / 32 + 1;
            std::vector<uint32_t> w(nw, 0);
            if (c.polyA > 0)
                for (int i = std::max(fullLen - 25 + 1, 0); i < fullLen; ++i) w[i / 32] |= (1u << (i % 32));
            for (int i = 0; i < nw; ++i) fprintf(f, "%u%c", w[i], i + 1 < nw ? ' ' : '\n');
        }
        fclose(f);
        f = xopen(c.out + "/ref/r.ti");
        if (!c.genome) {
            fprintf(f, "%d 1\n", c.M);
            for (int t = 1; t <= c.M; ++t)
                fprintf(f, "T%d\nG%d\nT%d\n+ %d\n1 1 %d\n\n", t, fam_of[t] + 1, t, (int)tseq[t].size(), (int)tseq[t].size());
        } else {
            // genome mode: four families per chromosome, each a locus on a random strand.  An isoform is its unique
            // prefix as one exon plus the shared body cut into 1-4 exons, with introns between; a read from the body
            // therefore lands on the same genomic alignment from every isoform.  On '-' the transcript's 5' end is its
            // highest coordinate: the body exons come first in the genome, the prefixes after them.
            Rng gg(c.seed ^ 0x67656e6f6d65ull);
            std::vector<std::vector<std::pair<int, int>>> ex(c.M + 1);
            std::vector<int> chr_of(c.M + 1), chr_len;
            std::vector<char> strand(c.M + 1);
            int cursor = 0;
            for (int fi = 0; fi < F; ++fi) {
                if (fi % 4 == 0) { if (fi) chr_len.push_back(cursor + 1000); cursor = 1000; }
                const int t0 = fam_start[fi], t1 = fam_start[fi + 1];
                const int blen = (int)body[fi].size();
                const char sd = gg.below(2) ? '-' : '+';
                std::vector<int> cuts;   // body part boundaries in transcript order
                const int parts = 1 + gg.below(4);
                for (int k = 1; k < parts; ++k) cuts.push_back(gg.range(20, blen - 20));
                std::sort(cuts.begin(), cuts.end());
                cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
                cuts.insert(cuts.begin(), 0);
                cuts.push_back(blen);
                std::vector<std::pair<int, int>> body_ex, pre_ex(c.M + 1, {0, 0});
                auto place_body = [&]() {
                    const int n = (int)cuts.size() - 1;
                    std::vector<std::pair<int, int>> e(n);
                    for (int k = 0; k < n; ++k) {   // genomic order: transcript order on '+', reversed on '-'
                        const int part = sd == '+' ? k : n - 1 - k;
                        const int len = cuts[part + 1] - cuts[part];
                        e[k] = {cursor + 1, cursor + len};
                        cursor += len + gg.range(50, 2000);
                    }
                    body_ex = e;
                };
                auto place_prefixes = [&]() {
                    for (int t = t0; t < t1; ++t)
                        if (prefix_len[t] > 0) {
                            pre_ex[t] = {cursor + 1, cursor + prefix_len[t]};
                            cursor += prefix_len[t] + gg.range(50, 2000);
                        }
                };
                if (sd == '+') { place_prefixes(); place_body(); }
                else { place_body(); place_prefixes(); }
                for (int t = t0; t < t1; ++t) {
                    std::vector<std::pair<int, int>> e = body_ex;
                    if (prefix_len[t] > 0) {
                        if (sd == '+') e.insert(e.begin(), pre_ex[t]);
                        else e.push_back(pre_ex[t]);
                    }
                    ex[t] = e;
                    chr_of[t] = (int)chr_len.size() + 1;
                    strand[t] = sd;
                }
            }
            chr_len.push_back(cursor + 1000);
            fprintf(f, "%d 0\n", c.M);
            for (int t = 1; t <= c.M; ++t) {
                fprintf(f, "T%d\nG%d\nchr%d\n%c %d\n%d", t, fam_of[t] + 1, chr_of[t], strand[t], (int)tseq[t].size(), (int)ex[t].size());
                for (auto& e : ex[t]) fprintf(f, " %d %d", e.first, e.second);
                fprintf(f, "\n\n");
            }
            FILE* fc = xopen(c.out + "/ref/r.chrlist");
            for (size_t k = 0; k < chr_len.size(); ++k) fprintf(fc, "chr%zu\t%d\n", k + 1, chr_len[k]);
            fclose(fc);
        }
        fclose(f);
        f = xopen(c.out + "/ref/r.grp");
        for (int s : fam_start) fprintf(f, "%d\n", s);
        fclose(f);
        f = xopen(c.out + "/s.temp/s.omit");
        for (int t = Mhit + 1; t <= c.M; ++t) fprintf(f, "%d\n", t);
        fclose(f);
    }

    // ---- expression weights --------------------------------------------------------------
    if (c.has_sample_seed) g = Rng(c.sample_seed);
    std::vector<double> fam_cdf(F);
    int Fhit = 0;
    {
        double a = 0;
        for (int f = 0; f < F; ++f) {
            bool hittable = fam_start[f] <= Mhit;
            if (c.expressed_frac < 1.0 && f > 0 && g.uni() >= c.expressed_frac) hittable = false;   // family 0 stays expressed
            double u = g.uni();
            a += hittable ? u * u * u * u + 1e-6 : 0.0;
            fam_cdf[f] = a;
            if (hittable) Fhit = f + 1;
        }
        for (auto& x : fam_cdf) x /= a;
    }
    std::vector<double> member_w(c.M + 1);
    for (int t = 1; t <= c.M; ++t) member_w[t] = 0.05 + g.uni();

    // ---- reads ------------------------------------------------------------------------------
    const char* ext = hasQ ? "fq" : "fa";
    FILE *fr[2] = {nullptr, nullptr}, *fu[2] = {nullptr, nullptr};
    if (paired) {
        fr[0] = xopen(c.out + "/s.temp/s_alignable_1." + ext); fr[1] = xopen(c.out + "/s.temp/s_alignable_2." + ext);
        if (c.N0 > 0) { fu[0] = xopen(c.out + "/s.temp/s_un_1." + ext); fu[1] = xopen(c.out + "/s.temp/s_un_2." + ext); }
    } else {
        fr[0] = xopen(c.out + "/s.temp/s_alignable." + ext);
        if (c.N0 > 0) fu[0] = xopen(c.out + "/s.temp/s_un." + ext);
    }
    auto put = [&](FILE* f, const char* tag, long id, int mate, const std::string& s, const std::string& q) {
        if (hasQ) fprintf(f, "@%s%ld/%d\n%s\n+\n%s\n", tag, id, mate, s.c_str(), q.c_str());
        else fprintf(f, ">%s%ld/%d\n%s\n", tag, id, mate, s.c_str());
    };

    FILE* fsam = nullptr;
    if (c.sam) {
        fsam = xopen(c.out + "/aln.sam");
        fprintf(fsam, "@HD\tVN:1.0\tSO:unsorted\n");
        for (int t = 1; t <= c.M; ++t) fprintf(fsam, "@SQ\tSN:T%d\tLN:%d\n", t, (int)tseq[t].size() + c.polyA);
        fprintf(fsam, "@PG\tID:gen_dataset\n");
    }
    // .dat body goes to a temp buffer file first because the header needs nHits
    std::string datp = c.out + "/s.temp/s.dat";
    FILE* fd = xopen(datp + ".body");
    uint64_t nHits = 0;
    std::vector<Hit> hits;
    std::string s1, q1, s2, q2;
    for (long r = 0; r < c.N1; ++r) {
        int f = (int)(std::lower_bound(fam_cdf.begin(), fam_cdf.begin() + Fhit, g.uni()) - fam_cdf.begin());
        if (f >= Fhit) f = Fhit - 1;
        int t0 = fam_start[f], t1 = std::min(fam_start[f + 1], Mhit + 1);  // members [t0, t1)
        // member of origin by within-family weight
        double tw = 0; for (int t = t0; t < t1; ++t) tw += member_w[t];
        double u = g.uni() * tw; int src = t0;
        for (int t = t0; t < t1; ++t) { u -= member_w[t]; src = t; if (u < 0) break; }
        int L1 = c.read_len - (c.var_len > 0 ? g.below(c.var_len + 1) : 0);
        int L2 = c.read_len - (c.var_len > 0 ? g.below(c.var_len + 1) : 0);
        int flen = paired ? std::max(g.range(c.frag_min, c.frag_max), std::max(L1, L2)) : L1;
        int slen = (int)tseq[src].size();
        if (flen > slen) flen = slen;
        int fpos = g.below(slen - flen + 1);           // forward-strand start on the source transcript
        int dir = g.uni() < c.probF ? 0 : 1;
        hits.clear();
        int boff = fpos - prefix_len[src];             // offset inside the shared body (may be < 0)
        for (int t = t0; t < t1; ++t) {
            int p;
            if (t == src) p = fpos;
            else if (boff >= 0) p = prefix_len[t] + boff;   // entirely inside the body -> every member
            else continue;
            int totLen = (int)tseq[t].size() + c.polyA;
            int pos = dir == 0 ? p : totLen - p - flen;     // strand-local coordinate
            hits.push_back({dir == 0 ? t : -t, pos, flen, p});
        }
        std::string frag = tseq[src].substr(fpos, flen);
        if (dir == 1) frag = revcomp(frag);
        sequence(g, frag.substr(0, L1), c.nfrac, s1, q1);
        if (paired) sequence(g, revcomp(frag).substr(0, L2), c.nfrac, s2, q2);
        if (c.spurious > 0 && g.uni() < c.spurious) {       // one random extra hit (junk alignment)
            int t = 1 + g.below(Mhit);
            int totLen = (int)tseq[t].size() + c.polyA;
            if (flen <= (int)tseq[t].size()) {
                int d2 = g.below(2);
                int p = g.below((int)tseq[t].size() - flen + 1);
                hits.push_back({d2 == 0 ? t : -t, d2 == 0 ? p : totLen - p - flen, flen, p});
            }
        }
        fprintf(fd, "%zu", hits.size());
        for (auto& h : hits) {
            if (paired) fprintf(fd, " %d %d %d", h.sid, h.pos, h.insertL);
            else fprintf(fd, " %d %d", h.sid, h.pos);
        }
        fputc('\n', fd);
        nHits += hits.size();
        put(fr[0], "r", r, 1, s1, q1);
        if (paired) put(fr[1], "r", r, 2, s2, q2);
        if (fsam) {  // all alignments of a read adjacent; reverse-strand records carry the reverse complement (SAM convention)
            const std::string rs1 = revcomp(s1), rq1(q1.rbegin(), q1.rend()), rs2 = paired ? revcomp(s2) : std::string(),
                              rq2 = paired ? std::string(q2.rbegin(), q2.rend()) : std::string();
            for (auto& h : hits) {
                const int t = std::abs(h.sid);
                const bool rev = h.sid < 0;
                if (!paired) {
                    fprintf(fsam, "r%ld\t%d\tT%d\t%d\t255\t%dM\t*\t0\t0\t%s\t%s\n", r, rev ? 16 : 0, t, h.fwd + 1, L1,
                            rev ? rs1.c_str() : s1.c_str(), hasQ ? (rev ? rq1.c_str() : q1.c_str()) : "*");
                } else {
                    const int p1 = rev ? h.fwd + h.insertL - L1 + 1 : h.fwd + 1;  // mate 1: 1-based leftmost forward coordinate
                    const int p2 = rev ? h.fwd + 1 : h.fwd + h.insertL - L2 + 1;
                    fprintf(fsam, "r%ld\t%d\tT%d\t%d\t255\t%dM\t=\t%d\t%d\t%s\t%s\n", r, rev ? 83 : 99, t, p1, L1, p2,
                            rev ? -h.insertL : h.insertL, rev ? rs1.c_str() : s1.c_str(), hasQ ? (rev ? rq1.c_str() : q1.c_str()) : "*");
                    fprintf(fsam, "r%ld\t%d\tT%d\t%d\t255\t%dM\t=\t%d\t%d\t%s\t%s\n", r, rev ? 163 : 147, t, p2, L2, p1,
                            rev ? h.insertL : -h.insertL, rev ? s2.c_str() : rs2.c_str(), hasQ ? (rev ? q2.c_str() : rq2.c_str()) : "*");
                }
            }
        }
    }
    fclose(fd);
    for (long r = 0; r < c.N0; ++r) {   // unalignable (noise) reads
        int L1 = c.read_len - (c.var_len > 0 ? g.below(c.var_len + 1) : 0);
        sequence(g, randseq(g, L1), c.nfrac, s1, q1);
        put(fu[0], "u", r, 1, s1, q1);
        if (paired) {
            int L2 = c.read_len - (c.var_len > 0 ? g.below(c.var_len + 1) : 0);
            sequence(g, randseq(g, L2), c.nfrac, s2, q2);
            put(fu[1], "u", r, 2, s2, q2);
        }
        if (fsam) {
            if (!paired) fprintf(fsam, "u%ld\t4\t*\t0\t0\t*\t*\t0\t0\t%s\t%s\n", r, s1.c_str(), hasQ ? q1.c_str() : "*");
            else {
                fprintf(fsam, "u%ld\t77\t*\t0\t0\t*\t*\t0\t0\t%s\t%s\n", r, s1.c_str(), hasQ ? q1.c_str() : "*");
                fprintf(fsam, "u%ld\t141\t*\t0\t0\t*\t*\t0\t0\t%s\t%s\n", r, s2.c_str(), hasQ ? q2.c_str() : "*");
            }
        }
    }
    if (fsam) fclose(fsam);
    for (int i = 0; i < 2; ++i) { if (fr[i]) fclose(fr[i]); if (fu[i]) fclose(fu[i]); }

    {   // .dat = 100-char padded header + body (parseIt.cpp:197-211)
        FILE* f = xopen(datp);
        char hdr[128];
        int n = snprintf(hdr, sizeof hdr, "%ld %llu %d", c.N1, (unsigned long long)nHits, c.read_type);
        fputs(hdr, f);
        for (int i = n; i < 100; ++i) fputc(' ', f);
        fputc('\n', f);
        FILE* b = fopen((datp + ".body").c_str(), "r");
        std::vector<char> buf(1 << 20);
        size_t k;
        while ((k = fread(buf.data(), 1, buf.size(), b)) > 0) fwrite(buf.data(), 1, k, f);
        fclose(b); fclose(f);
        remove((datp + ".body").c_str());
    }
    {
        FILE* f = xopen(c.out + "/s.stat/s.cnt");
        fprintf(f, "%ld %ld 0 %ld\n", c.N0, c.N1, c.N0 + c.N1);
        fclose(f);
        f = xopen(c.out + "/s.temp/s.mparams");
        fprintf(f, "%d %d\n%.10g\n%d\n%d\n%d %d\n%.10g %.10g\n%d\n", c.minL, c.maxL, c.probF, c.est_rspd, c.B, 1, c.maxL,
                c.frag_mean, c.frag_sd, c.seed_len);
        fclose(f);
    }
    fprintf(stderr, "gen_dataset: M=%d families=%d N1=%ld N0=%ld nHits=%llu read_type=%d -> %s\n", c.M, F, c.N1, c.N0,
            (unsigned long long)nHits, c.read_type, c.out.c_str());
    return 0;
}
