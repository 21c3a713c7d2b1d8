// rsem-b200-host-selftest: runs the multi-threaded host parsers / formatters of the drop-in executables without a
// GPU and dumps what they produced as raw binary arrays, so that the CPU test suite can compare them with an
// independent parse of the same text files and across thread counts.  Test tooling, not part of the product path.
//
//   rsem-b200-host-selftest <imdName> <read_type> <threads> <seedLen> <outPrefix>
//
// writes <outPrefix>.{row_ptr.u64,sid.i32,pos.i32,insertL.i32,off<m>.u64,base<m>.u8,qual<m>.u8,lowq.u8} and
// <outPrefix>.ofg (write_ofg of a synthetic conprb) plus the arrays load_ofg reads back from it.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "host.hpp"

using namespace host;

template <class T>
static void dump(const std::string& path, const std::vector<T>& v) {
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) die("cannot write " + path);
    if (!v.empty() && fwrite(v.data(), sizeof(T), v.size(), f) != v.size()) die("short write " + path);
    fclose(f);
}

// rsem-b200-host-selftest --bam-copy in.(sam|bam) out.bam threads [weight_step]
// reads every record with AlnReader and writes it with BamWriter; with weight_step > 0 the k-th mapped record gets the
// posterior (k * weight_step) mod 1 through set_alignment_weight (MAPQ + ZW:f), like rsem-run-em -b does.
static int bam_copy(int argc, char** argv) {
    if (argc < 5) { fprintf(stderr, "Usage: rsem-b200-host-selftest --bam-copy in out.bam threads [weight_step]\n"); return -1; }
    const double step = argc > 5 ? atof(argv[5]) : 0.0;
    AlnReader in(argv[2]);
    BamWriter out(argv[3], rsem_bam_header_text(in.header_text()), atoi(argv[4]));
    BamRecord r;
    unsigned long long n = 0, mapped = 0;
    while (in.next(r)) {
        ++n;
        if (step > 0 && r.mapped()) {
            ++mapped;
            r.set_alignment_weight(std::fmod((double)mapped * step, 1.0));
        }
        out.write(r);
    }
    out.close();
    printf("records %llu mapped %llu refs %zu\n", n, mapped, in.ref_names().size());
    return 0;
}

// rsem-b200-host-selftest --bam-sort in.(sam|bam) out.bam threads
// a stable in-memory sort of every record by (tid, pos), records without a target last, as `samtools sort` orders a
// BAM by coordinate; the benchmark and the tests of rsem-bam2wig / rsem-bam2readdepth sort their inputs with it
static int bam_sort(int argc, char** argv) {
    if (argc != 5) { fprintf(stderr, "Usage: rsem-b200-host-selftest --bam-sort in out.bam threads\n"); return -1; }
    g_io_threads = std::max(1, atoi(argv[4]));
    AlnReader in(argv[2]);
    std::vector<uint8_t> data;
    std::vector<std::pair<uint64_t, uint64_t>> keys;   // (tid, pos) key, offset of the record's block_size
    BamRecord r;
    while (in.next(r)) {
        const int32_t tid = r.tid();
        const uint64_t k = tid < 0 ? ~0ull : ((uint64_t)(uint32_t)tid << 32) | (uint32_t)(r.pos() + 1);
        keys.emplace_back(k, data.size());
        const uint32_t n = (uint32_t)r.data.size();
        const uint8_t b4[4] = {(uint8_t)n, (uint8_t)(n >> 8), (uint8_t)(n >> 16), (uint8_t)(n >> 24)};
        data.insert(data.end(), b4, b4 + 4);
        data.insert(data.end(), r.data.begin(), r.data.end());
    }
    std::stable_sort(keys.begin(), keys.end(), [](const std::pair<uint64_t, uint64_t>& a, const std::pair<uint64_t, uint64_t>& b) {
        return a.first < b.first;
    });
    BamWriter out(argv[3], rsem_bam_header_text(in.header_text()), g_io_threads);
    std::vector<uint8_t> buf;
    for (const auto& k : keys) {
        const uint8_t* p = data.data() + k.second;
        const size_t n = 4 + (p[0] | (p[1] << 8) | (p[2] << 16) | ((size_t)p[3] << 24));
        buf.insert(buf.end(), p, p + n);
        if (buf.size() >= (64u << 20)) { out.write_encoded(buf.data(), buf.size()); buf.clear(); }
    }
    if (!buf.empty()) out.write_encoded(buf.data(), buf.size());
    out.close();
    printf("records %zu\n", keys.size());
    return 0;
}

// rsem-b200-host-selftest --wig-format wig|depth chunk_positions threads values.f64 out length...
// format_wiggles on targets t0, t1, ... whose values are read one after another from values.f64 (native doubles); a
// length written as eN is a target of length N with the reference's empty read_depth
static int wig_format(int argc, char** argv) {
    if (argc < 8) { fprintf(stderr, "Usage: rsem-b200-host-selftest --wig-format wig|depth chunk threads values.f64 out length...\n"); return -1; }
    const bool wig = std::string(argv[2]) == "wig";
    const std::vector<char> raw = slurp(argv[5]);
    std::vector<double> v(raw.size() / 8);
    if (!v.empty()) memcpy(v.data(), raw.data(), v.size() * 8);
    std::vector<WigTarget> ts;
    size_t at = 0;
    for (int i = 7; i < argc; ++i) {
        WigTarget t;
        t.name = "t" + std::to_string(i - 7);
        const bool empty = argv[i][0] == 'e';
        t.length = strtoull(argv[i] + (empty ? 1 : 0), nullptr, 10);
        if (!empty && t.length) {
            if (at + t.length > v.size()) die("--wig-format: not enough values");
            t.depth = v.data() + at;
            at += t.length;
        }
        ts.push_back(t);
    }
    std::vector<std::string> chunks;
    format_wiggles(ts, wig, strtoull(argv[3], nullptr, 10), atoi(argv[4]), chunks);
    FILE* f = fopen(argv[6], "wb");
    if (!f) die(std::string("cannot write ") + argv[6]);
    for (const std::string& c : chunks) fwrite(c.data(), 1, c.size(), f);
    fclose(f);
    printf("chunks %zu\n", chunks.size());
    return 0;
}

// rsem-b200-host-selftest --sidecar imdName read_type threads seedLen has_polyA outPrefix
// loads imdName.b200 (written by bin/rsem-parse-alignments) the way rsem-run-em does and dumps the same arrays as the text
// mode below (hits + the alignable read set with its lowq flags), plus the number / first names of the short reads.
static int sidecar_dump(int argc, char** argv) {
    if (argc != 8) { fprintf(stderr, "Usage: rsem-b200-host-selftest --sidecar imdName read_type threads seedLen has_polyA outPrefix\n"); return -1; }
    const std::string imd = argv[2], out = argv[7];
    const int read_type = atoi(argv[3]);
    g_io_threads = atoi(argv[4]);
    const int seed_len = atoi(argv[5]);
    const bool has_polyA = atoi(argv[6]) != 0;
    g_verbose = false;
    Sidecar sc;
    if (!load_sidecar(imd, read_type, sc)) { printf("no usable side-car\n"); return 3; }
    dump(out + ".row_ptr.u64", sc.hits.row_ptr);
    dump(out + ".sid.i32", sc.hits.sid);
    dump(out + ".pos.i32", sc.hits.pos);
    dump(out + ".insertL.i32", sc.hits.insertL);
    unsigned long long n_short_tot = 0;
    for (int tag = 0; tag < 3; ++tag) {
        ReadStore& rs = sc.reads[tag];
        std::vector<std::string> names;
        uint64_t n_short = 0;
        finish_sidecar_reads(rs, sc.shorts[tag], has_polyA, seed_len, &names, &n_short);
        n_short_tot += n_short;
        const std::string pre = out + (tag == 1 ? "" : (tag == 0 ? ".un" : ".max"));
        for (int m = 0; m < rs.n_mates; ++m) {
            dump(pre + ".off" + std::to_string(m) + ".u64", rs.off[m]);
            dump(pre + ".base" + std::to_string(m) + ".u8", rs.base[m]);
            dump(pre + ".qual" + std::to_string(m) + ".u8", rs.qual[m]);
        }
        dump(pre + ".lowq.u8", rs.lowq);
        for (const std::string& nm : names) printf("short %d %s\n", tag, nm.c_str());
    }
    printf("N %llu H %llu reads %llu %llu %llu short %llu\n", (unsigned long long)sc.hits.N, (unsigned long long)sc.hits.H,
           (unsigned long long)sc.reads[0].n, (unsigned long long)sc.reads[1].n, (unsigned long long)sc.reads[2].n, n_short_tot);
    return 0;
}

// rsem-b200-host-selftest --mapq-table: the MAPQ threshold table rsem-tbam2gbam hands to the device against
// prb_to_mapq for every float in [0, 2]; prints the number of floats checked and of mismatches
static int mapq_table() {
    const std::vector<float> t = mapq_thresholds();
    const uint32_t hi = 0x40000000u;   // 2.0f
    const int T = std::max(1u, std::thread::hardware_concurrency());
    std::vector<uint64_t> bad(T, 0);
    std::vector<std::thread> pool;
    for (int k = 0; k < T; ++k)
        pool.emplace_back([&, k]() {
            for (uint64_t bits = k; bits <= hi; bits += T) {
                float p;
                const uint32_t b32 = (uint32_t)bits;
                memcpy(&p, &b32, 4);
                int m = 0;
                for (int j = 1; j <= 100; ++j) m += p >= t[j];
                if (m != prb_to_mapq(p)) ++bad[k];
            }
        });
    for (auto& th : pool) th.join();
    uint64_t nbad = 0;
    for (uint64_t b : bad) nbad += b;
    printf("%llu floats, %llu mismatches\n", (unsigned long long)hi + 1, (unsigned long long)nbad);
    return nbad ? 1 : 0;
}

// rsem-b200-host-selftest --ti ref.ti: load_transcripts' fields, one transcript per line, tab-separated:
// id, name, gene id, gene name, seqname, strand, length, exon length sum, then start-end of every exon
static int ti_dump(const char* path) {
    std::vector<TranscriptInfo> tr;
    int type = -1;
    load_transcripts(path, tr, &type);
    printf("%d %d\n", (int)tr.size() - 1, type);
    for (size_t i = 1; i < tr.size(); ++i) {
        const TranscriptInfo& t = tr[i];
        printf("%s\t%s\t%s\t%s\t%s\t%c\t%d\t%d", t.transcript_id.c_str(), t.transcript_name.c_str(), t.gene_id.c_str(),
               t.gene_name.c_str(), t.seqname.c_str(), t.strand, t.length, t.exon_length);
        for (auto& e : t.exons) printf("\t%d-%d", e.first, e.second);
        printf("\n");
    }
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 2 && std::string(argv[1]) == "--mapq-table") return mapq_table();
    if (argc >= 3 && std::string(argv[1]) == "--ti") return ti_dump(argv[2]);
    if (argc >= 2 && std::string(argv[1]) == "--bam-copy") return bam_copy(argc, argv);
    if (argc >= 2 && std::string(argv[1]) == "--sidecar") return sidecar_dump(argc, argv);
    if (argc >= 2 && std::string(argv[1]) == "--bam-sort") return bam_sort(argc, argv);
    if (argc >= 2 && std::string(argv[1]) == "--wig-format") return wig_format(argc, argv);
    if (argc != 6) {
        fprintf(stderr, "Usage: rsem-b200-host-selftest imdName read_type threads seedLen outPrefix\n");
        return -1;
    }
    const std::string imd = argv[1], out = argv[5];
    const int read_type = atoi(argv[2]);
    g_io_threads = atoi(argv[3]);
    const int seed_len = atoi(argv[4]);
    g_verbose = false;

    unsigned long long n1 = 0;
    {
        FILE* f = fopen((imd + ".dat").c_str(), "r");
        if (!f || fscanf(f, "%llu", &n1) != 1) die("cannot read " + imd + ".dat");
        fclose(f);
    }
    HitStore h;
    load_dat(imd + ".dat", read_type, n1, h);
    dump(out + ".row_ptr.u64", h.row_ptr);
    dump(out + ".sid.i32", h.sid);
    dump(out + ".pos.i32", h.pos);
    dump(out + ".insertL.i32", h.insertL);

    ReadStore rs;
    std::vector<std::string> short_names;
    uint64_t n_short = 0;
    parse_reads(imd, 1, read_type, false, seed_len, rs, &short_names, &n_short);
    for (int m = 0; m < rs.n_mates; ++m) {
        dump(out + ".off" + std::to_string(m) + ".u64", rs.off[m]);
        dump(out + ".base" + std::to_string(m) + ".u8", rs.base[m]);
        dump(out + ".qual" + std::to_string(m) + ".u8", rs.qual[m]);
    }
    dump(out + ".lowq.u8", rs.lowq);

    // .ofg round trip on a synthetic matrix derived from the hit indices (includes dropped entries and rows)
    std::vector<double> conprb(h.H), ncpv(h.N);
    for (uint64_t j = 0; j < h.H; ++j) {
        const uint64_t x = j * 2654435761ull % 1000003ull;
        conprb[j] = x % 17 == 0 ? 0.0 : std::pow(10.0, -3.0 - (double)(x % 290)) * (1.0 + (double)(x % 97) / 97.0);
    }
    for (uint64_t i = 0; i < h.N; ++i) {
        const uint64_t x = i * 40503ull % 65521ull;
        ncpv[i] = x % 5 == 0 ? 0.0 : std::pow(10.0, -40.0 - (double)(x % 200));
    }
    int M = 0;
    for (int32_t s : h.sid) M = std::max(M, std::abs(s));
    write_ofg(out + ".ofg", M, 12345, h, conprb, ncpv);
    uint64_t n0 = 0;
    std::vector<uint64_t> rp;
    std::vector<int32_t> sid;
    std::vector<double> con;
    load_ofg(out + ".ofg", M, n0, rp, sid, con, false);   // the text
    {   // and the binary side-car write_ofg left next to it: must be the very same arrays
        uint64_t n0b = 0;
        std::vector<uint64_t> rp2;
        std::vector<int32_t> sid2;
        std::vector<double> con2;
        load_ofg(out + ".ofg", M, n0b, rp2, sid2, con2, true);
        const bool same = n0b == n0 && rp2 == rp && sid2 == sid && con2.size() == con.size() &&
                          (con.empty() || !memcmp(con2.data(), con.data(), con.size() * sizeof(double)));
        FILE* sf = fopen((out + ".ofg.b200").c_str(), "rb");
        printf("ofg_sidecar present %d identical %d\n", sf ? 1 : 0, same ? 1 : 0);
        if (sf) fclose(sf);
    }
    dump(out + ".ofg_row_ptr.u64", rp);
    dump(out + ".ofg_sid.i32", sid);
    dump(out + ".ofg_con.f64", con);
    dump(out + ".in_con.f64", conprb);
    dump(out + ".in_ncpv.f64", ncpv);
    printf("N %llu H %llu reads %llu short %llu N0 %llu ofg_rows %zu ofg_entries %zu\n", (unsigned long long)h.N,
           (unsigned long long)h.H, (unsigned long long)rs.n, (unsigned long long)n_short, (unsigned long long)n0,
           rp.empty() ? (size_t)0 : rp.size() - 1, sid.size());
    return 0;
}
