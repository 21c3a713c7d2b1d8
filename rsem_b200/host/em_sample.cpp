// Per-sample output stages of rsem-run-em, shared by rsem-run-em and rsem-run-em-batch.
#include <cstdlib>
#include <ctime>

#include "host.hpp"

namespace host {

// EM.cpp:504-536 + BamWriter::work (BamWriter.h:82-146): every mapped alignment line (pair of lines for paired-end
// reads) takes the next hit's posterior, in .dat order; all lines are written back, mates with read 1 first.
void write_posterior_bam(const std::string& inpSamF, const std::string& outName, int read_type, bool sampling, bool hasSeed,
                         uint32_t seed, const std::vector<TranscriptInfo>& tr, int ti_type, const HitStore& hits,
                         std::vector<double>& post, const std::vector<double>& post0, int threads, bool verbose) {
    if (sampling) {  // one alignment (or the noise entry) per read, drawn from its posterior (EM.cpp:507-531)
        Mt engine(hasSeed ? seed : (uint32_t)time(NULL));
        if (verbose) printf("Begin to sample reads from their posteriors.\n");
        std::vector<double> arr;
        for (uint64_t j = 0; j < hits.N; ++j) {
            const uint64_t fr = hits.row_ptr[j], to = hits.row_ptr[j + 1];
            const int len = (int)(to - fr + 1);
            arr.assign(len, 0.0);
            arr[0] = post0[j];
            for (uint64_t k = fr; k < to; ++k) arr[k - fr + 1] = arr[k - fr] + post[k];
            int id = -1;
            if (!(arr[len - 1] < kEps)) {  // sample(): first index with arr[index] > u * total (sampling.h:50-65)
                const double prb = engine.uniform01() * arr[len - 1];
                int l = 0, r = len - 1;
                while (l <= r) {
                    const int mid = (l + r) / 2;
                    if (arr[mid] <= prb) l = mid + 1;
                    else r = mid - 1;
                }
                if (l >= len) die("sampling: the draw fell outside the cumulative posterior (reference: assert(l < len))");
                id = l;
            }
            for (uint64_t k = fr; k < to; ++k) post[k] = ((int)(k - fr + 1) == id ? 1.0 : 0.0);
        }
        if (verbose) printf("Sampling is finished.\n");
    }
    AlnReader in(inpSamF);
    const std::vector<int> e2i = map_bam_targets(in.ref_names(), tr, ti_type);
    BamWriter out(outName + ".transcript.bam", rsem_bam_header_text(in.header_text()), threads);
    const bool paired = read_type >= 2;
    uint64_t next_hit = 0, cnt = 0;
    auto take_hit = [&](const BamRecord& b) {
        if (next_hit >= hits.H) die("The alignment file has more aligned lines than the .dat file has alignments (reference: assert(hit != NULL))!");
        const int32_t t = b.tid();
        if (t < 0 || t >= (int32_t)e2i.size() || e2i[t] != std::abs(hits.sid[next_hit]))
            die("The alignment file does not match the .dat file (reference: assert(getInternalSid(tid + 1) == hit->getSid()))!");
        return post[next_hit++];
    };
    BamRecord b, b2;
    if (!paired) {
        while (in.next(b)) {
            ++cnt;
            if (verbose && cnt % 1000000 == 0) printf("%llu alignment lines are loaded!\n", (unsigned long long)cnt);
            if (b.mapped()) b.set_alignment_weight(take_hit(b));
            out.write(b);
        }
    } else {
        while (in.next(b) && in.next(b2)) {
            cnt += 2;
            if (verbose && cnt % 1000000 == 0) printf("%llu alignment lines are loaded!\n", (unsigned long long)cnt);
            if (!b.read1()) b.data.swap(b2.data);
            if (b.mapped() && b2.mapped()) {
                const double w = take_hit(b);
                if (b2.tid() != b.tid()) die("The two mates of a read pair align to different transcripts in the alignment file!");
                b.set_alignment_weight(w);
                b2.set_alignment_weight(w);
            }
            out.write(b);
            out.write(b2);
        }
    }
    if (next_hit != hits.H) die("The alignment file has fewer aligned lines than the .dat file has alignments (reference: assert(wrapper.getNextHit() == NULL))!");
    out.close();
    if (verbose) printf("Bam output file is generated!\n");
}


// .theta (EM.cpp:484-500), .model and the result rows (EM.cpp:480-502); counts[0] already holds N0
void write_em_outputs(const std::string& refName, const std::string& imdName, const std::string& statName,
                      const RefData& refs, const std::vector<TranscriptInfo>& transcripts, const HostModel& model,
                      std::vector<double> theta, const std::vector<double>& counts, bool appendNames) {
    FILE* fo = fopen((statName + ".theta").c_str(), "w");
    if (!fo) die("Cannot open " + statName + ".theta for writing!");
    const int M = refs.M;
    std::vector<double> eel;
    fprintf(fo, "%d\n", M + 1);
    for (int i = 0; i < M; ++i) fprintf(fo, "%.15g ", theta[i]);
    fprintf(fo, "%.15g\n", theta[M]);
    calc_eel(refs, model.gld, eel);
    polish_theta(theta, eel, model.mw);
    for (int i = 0; i < M; ++i) fprintf(fo, "%.15g ", theta[i]);
    fprintf(fo, "%.15g\n", theta[M]);
    fclose(fo);
    model.write(statName + ".model");
    write_results_em(refName, imdName, transcripts, theta, eel, counts.data(), appendNames);
}

}  // namespace host
