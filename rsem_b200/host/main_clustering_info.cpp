// bin/rsem-for-ebseq-calculate-clustering-info: drop-in for the reference's tool of that name
// (EBSeq/calcClusteringInfo.cpp), the first step of rsem-generate-ngvector.
//
//   rsem-for-ebseq-calculate-clustering-info k input_reference_fasta_file output_file
//
// For every transcript t with effL_t = len_t - k + 1 > 0 the output line is name_t \t c_t / effL_t, where c_t counts the
// start positions of t whose k-mer also starts in another transcript; effL_t <= 0 gives -1 (:114-140).  The counts come
// from the device (K9, csrc/kmer_kernels.cu); stdout and the output file are the reference's, byte for byte.
//
// The FASTA is read the way loadRef (:61-90) reads it with getline, from one buffer in one pass: the tag is the whole
// header line after '>' (a trailing '\r' included), every following line not starting with '>' is appended (empty lines
// too), bases are upper-cased and every byte other than ACGT becomes N, and an entry with an empty sequence is dropped with
// the reference's warning.  A file whose first line does not start with '>' holds no transcripts.
//
// Without k-mer positions (every transcript shorter than k) there is no device work.  k <= 0 (atoi, :98) needs none
// either: the reference's comparator then compares no bases, so all positions form one group and every ratio is 1 when
// there are two or more transcripts, 0 when there is one.
//
// Differences: a missing or unreadable input is reported on stderr with exit status 255 and no output file (the reference
// aborts in an assert, :65); an output file that cannot be written is an error (the reference exits 0 without it).
// RSEM_B200_TIMING=1 prints the FASTA load time and the device time of each phase to stderr.
#include <algorithm>
#include <cerrno>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host.hpp"

using namespace host;

namespace {

struct Fasta {
    std::vector<std::string> names;
    std::vector<uint64_t> off{0};   // transcript t is bases[off[t] .. off[t + 1])
    std::vector<uint8_t> bases;     // 0 A, 1 C, 2 G, 3 T, 4 N
};

// the whole file, read to its end (pipes and process substitutions have no size to ask for)
std::vector<char> read_all(const char* path) {
    FILE* f = fopen(path, "rb");
    if (!f) die(std::string("Cannot open ") + path + "! It may not exist.");
    std::vector<char> buf;
    size_t used = 0;
    for (;;) {
        if (buf.size() - used < (1u << 20)) buf.resize(std::max<size_t>(2 * buf.size(), used + (1u << 20)));
        const size_t got = fread(buf.data() + used, 1, buf.size() - used, f);
        used += got;
        if (got == 0) break;
    }
    const bool failed = ferror(f);
    const int err = errno;
    fclose(f);
    if (failed) die(std::string("Cannot read ") + path + ": " + strerror(err));
    buf.resize(used);
    return buf;
}

void load_fasta(const char* path, Fasta& fa) {
    const std::vector<char> buf = read_all(path);
    uint8_t code[256];
    memset(code, 4, sizeof code);
    code['A'] = code['a'] = 0;
    code['C'] = code['c'] = 1;
    code['G'] = code['g'] = 2;
    code['T'] = code['t'] = 3;
    fa.bases.reserve(buf.size());
    const char* p = buf.data();
    const char* const end = p + buf.size();
    // getline: the line up to the next '\n'; the last line needs no '\n'; nothing after a final '\n' is a line
    auto next_line = [&](const char*& b, const char*& e) {
        if (p == end) return false;
        b = p;
        e = static_cast<const char*>(memchr(p, '\n', (size_t)(end - p)));
        if (!e) e = end;
        p = e == end ? end : e + 1;
        return true;
    };
    const char *b = nullptr, *e = nullptr;
    bool have = next_line(b, e);
    while (have && e > b && *b == '>') {
        std::string tag(b + 1, e);
        const size_t start = fa.bases.size();
        while ((have = next_line(b, e)) && !(e > b && *b == '>'))
            for (const char* c = b; c < e; ++c) fa.bases.push_back(code[(uint8_t)*c]);
        if (fa.bases.size() == start) {
            printf("Warning: Fasta entry %s has an empty sequence! It is omitted!\n", tag.c_str());
            continue;
        }
        fa.names.push_back(std::move(tag));
        fa.off.push_back(fa.bases.size());
    }
    printf("The reference is loaded.\n");
}

}  // namespace

int main(int argc, char* argv[]) {
    if (argc != 4) {
        printf("Usage: rsem-for-ebseq-calculate-clustering-info k input_reference_fasta_file output_file\n");
        exit(-1);
    }
    const int k = atoi(argv[1]);
    auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = now();
    Fasta fa;
    load_fasta(argv[2], fa);
    const double t1 = now();
    const size_t M = fa.names.size();

    // effL and the k-mer positions (:101-108), in 64 bits
    std::vector<int64_t> effL(M);
    uint64_t positions = 0;
    for (size_t t = 0; t < M; ++t) {
        effL[t] = std::max<int64_t>(0, (int64_t)(fa.off[t + 1] - fa.off[t]) - (int64_t)k + 1);
        positions += (uint64_t)effL[t];
    }
    printf("All possbile %d mers are generated.\n", k);

    std::vector<uint64_t> shared(M, 0);
    rsem_b200_kmer_stats st;
    memset(&st, 0, sizeof st);
    if (k <= 0) {
        if (M >= 2) for (size_t t = 0; t < M; ++t) shared[t] = (uint64_t)effL[t];
    } else if (positions > 0) {
        rsem_b200_ctx* ctx = nullptr;
        const char* dev = getenv("RSEM_B200_DEVICE");
        check_rc(rsem_b200_ctx_create(dev ? atoi(dev) : 0, &ctx), "ctx_create");
        rsem_b200_kmer_params kp;
        memset(&kp, 0, sizeof kp);
        kp.k = k;
        kp.n_transcripts = M;
        kp.offsets = fa.off.data();
        kp.bases = fa.bases.data();
        check_rc(rsem_b200_kmer_shared(ctx, &kp, shared.data(), &st), "kmer_shared");
        rsem_b200_ctx_destroy(ctx);
    }
    printf("All %d mers are sorted.\n", k);
    printf("Clustering information is calculated.\n");

    // name \t value with setprecision(6), i.e. %.6g (:139-141); names are written whole, NUL bytes included
    std::string out;
    out.reserve(M * 32);
    char num[64];
    for (size_t t = 0; t < M; ++t) {
        const double v = effL[t] == 0 ? -1.0 : (double)shared[t] / (double)effL[t];
        out += fa.names[t];
        out += '\t';
        out.append(num, (size_t)snprintf(num, sizeof num, "%.6g", v));
        out += '\n';
    }
    FILE* fo = fopen(argv[3], "wb");
    if (!fo) die(std::string("Cannot open ") + argv[3] + " for writing!");
    const bool ok = fwrite(out.data(), 1, out.size(), fo) == out.size();
    if (fclose(fo) != 0 || !ok) die(std::string("Cannot write ") + argv[3] + "!");
    if (getenv("RSEM_B200_TIMING"))
        fprintf(stderr,
                "rsem-for-ebseq-calculate-clustering-info timing: FASTA load %.3f s, total %.3f s; device: pack %.3f s, "
                "insert %.3f s, count %.3f s, %d passes, %llu positions, %llu table slots\n",
                t1 - t0, now() - t0, st.pack_ms / 1e3, st.insert_ms / 1e3, st.count_ms / 1e3, st.passes,
                (unsigned long long)positions, (unsigned long long)st.table_slots);
    return 0;
}
