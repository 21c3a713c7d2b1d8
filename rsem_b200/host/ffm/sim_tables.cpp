// The cumulative tables rsem-simulate-reads samples from (the startSimulation functions of the model classes) and the
// theta vector it derives from the results file (simulation.cpp:94-115).
//
// The reference compiles simulation.cpp with -O3 -ffast-math (Makefile:39,72-73); this file is built with the same
// flags and keeps the same operation order, so the tables hold the reference's bits: a different last bit in a
// cumulative array moves a binary-search boundary and changes the reads.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>
#include <vector>

#include "../host.hpp"

namespace host {

// theta[1..M] = TPM * eel normalised to 1 - theta[0]; TPM is the tab-separated column `offsite` after one header
// line.  Past the end of the file std::getline leaves `line` as it is once the stream is at EOF: a file whose last
// line ends without a newline repeats that line's TPM for every missing transcript; after a final newline the first
// missing line reads as empty (TPM 0) and so do the rest.  Returns the sum before normalising.
double sim_theta(const std::string& results_path, int M, int offsite, const std::vector<double>& eel,
                 std::vector<double>& theta) {
    std::ifstream fin(results_path.c_str());
    std::string line;
    double denom = 0.0;
    std::getline(fin, line);
    for (int i = 1; i <= M; i++) {
        std::getline(fin, line);
        size_t b = 0;
        for (int j = 0; j < offsite; j++) b = line.find_first_of('\t', b) + 1;
        size_t e = line.find_first_of('\t', b);
        if (e == std::string::npos) e = line.length();
        const double tpm = atof(line.substr(b, e - b).c_str());
        theta[i] = tpm * eel[i];
        denom += theta[i];
    }
    if (denom > kEps)
        for (int i = 1; i <= M; i++) theta[i] = theta[i] / denom * (1.0 - theta[0]);
    return denom;
}

void sim_prefix(const double* in, double* out, int n) {
    for (int i = 0; i < n; i++) {
        out[i] = in[i];
        if (i > 0) out[i] += out[i - 1];
    }
}

// (Q)Profile::startSimulation (QProfile.h:151-193, Profile.h:163-205): row prefix sums, then rows of a block that sum
// to 0 are replaced by the block's average match / N / other probabilities
void sim_profile_cdf(const std::vector<double>& p, int rows, std::vector<double>& pc) {
    const int NC = 5;
    pc.assign((size_t)rows * 25, 0.0);
    for (int i = 0; i < rows; i++) {
        const double* pi = &p[(size_t)i * 25];
        double* ci = &pc[(size_t)i * 25];
        for (int j = 0; j < NC; j++) sim_prefix(pi + j * NC, ci + j * NC, NC);
        double cp_sum = 0.0, cp_d = 0.0, cp_n = 0.0;
        for (int j = 0; j < NC - 1; j++) {
            cp_sum += ci[j * NC + NC - 1];
            cp_d += pi[j * NC + j];
            cp_n += pi[j * NC + NC - 1];
        }
        if (cp_sum == 0.0) continue;
        const double p_d = cp_d / cp_sum, p_n = cp_n / cp_sum;
        double p_o = (1.0 - p_d - p_n) / (NC - 2);
        for (int j = 0; j < NC - 1; j++) {
            if (ci[j * NC + NC - 1] > 0.0) continue;
            for (int k = 0; k < NC; k++) {
                ci[j * NC + k] = (k == j ? p_d : k == NC - 1 ? p_n : p_o);
                if (k > 0) ci[j * NC + k] += ci[j * NC + k - 1];
            }
        }
        if (ci[(NC - 1) * NC + NC - 1] == 0.0) {
            p_o = (1.0 - p_n) / (NC - 1);
            for (int k = 0; k < NC; k++) {
                ci[(NC - 1) * NC + k] = (k < NC - 1 ? p_o : p_n);
                if (k > 0) ci[(NC - 1) * NC + k] += ci[(NC - 1) * NC + k - 1];
            }
        }
    }
}

// NoiseQProfile::startSimulation (NoiseQProfile.h:153-166): a row that sums to ~0 samples A C G T uniformly
void sim_noiseq_cdf(const std::vector<double>& p, std::vector<double>& pc) {
    pc.assign(500, 0.0);
    for (int i = 0; i < 100; i++) {
        sim_prefix(&p[i * 5], &pc[i * 5], 5);
        if (std::fabs(pc[i * 5 + 4]) < 1e-8) {
            const double u[5] = {0.25, 0.5, 0.75, 1.0, 1.0};
            for (int j = 0; j < 5; j++) pc[i * 5 + j] = u[j];
        }
    }
}

// RSPD::startSimulation (RSPD.h:182-193): transcript i's evalCDF(j + 1, fullLen), j < fullLen, at off[i]
void sim_rspd_cdf(const std::vector<double>& pdf, const std::vector<double>& cdf, int B, const std::vector<int32_t>& full_len,
                  std::vector<uint64_t>& off, std::vector<double>& out) {
    const int M = (int)full_len.size() - 1;
    off.assign((size_t)M + 2, 0);
    for (int i = 1; i <= M; i++) off[i + 1] = off[i] + (uint64_t)full_len[i];
    out.assign(off[M + 1], 0.0);
    for (int i = 1; i <= M; i++) {
        const int fullLen = full_len[i];
        double* d = &out[off[i]];
        for (int j = 0; j < fullLen; j++) {
            const int fpos = j + 1;
            const int k = ((long long)fpos) * B / fullLen;
            const double val = fpos * 1.0 / fullLen * B;
            d[j] = cdf[k] + (val - k) * pdf[k + 1];
        }
    }
}

}  // namespace host
