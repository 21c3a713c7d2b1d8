// Phase I of rsem-calculate-credibility-intervals: nSpC theta vectors drawn from the Dirichlet posterior of every count
// vector of one count-vector file, each turned into a row of TPMs and its mean effective length (calcCI.cpp:93-164).
//
// Every draw is a Gamma variate from one mt19937 stream per file, accepted or rejected by comparing libm's tan / exp /
// log / pow against a uniform, so the host keeps this part: the device's libm differs from glibc in the last bit, and
// one flipped comparison shifts the rest of the stream.  The reference compiles calcCI.cpp with -O3 -ffast-math
// (Makefile:39,72-73); this file is built with the same flags.  The arithmetic below is written in the form gcc gives
// the reference under those flags (reciprocal multiplies for the divisions by a loop-invariant value, the float
// `tpm[] *= 1e6`, the float l_bar accumulated through a double add), so the rows carry the reference's bits whatever
// this compiler decides.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include "../host.hpp"

namespace host {

namespace {

// boost::random::uniform_01<double> on a 32-bit engine: one word, w * 2^-32
inline double uniform01(std::mt19937& eng) { return (uint32_t)eng() * 0x1p-32; }

// exponential_distribution(lambda = 1): -1 / lambda * log(1 - u)
inline double exponential(std::mt19937& eng) { return -std::log(1.0 - uniform01(eng)); }

// boost 1.55 gamma_distribution(alpha, beta = 1): alpha == 1 an exponential; alpha > 1 Cheng's rejection from a
// Cauchy proposal; alpha < 1 the Ahrens-Dieter GS algorithm.  `p` = e / (alpha + e) as the distribution stores it.
double gamma_draw(std::mt19937& eng, double alpha, double p) {
    if (alpha == 1.0) return exponential(eng);
    if (alpha > 1.0) {
        const double pi = 3.14159265358979323846;
        const double am1 = alpha - 1.0, s = std::sqrt(alpha + alpha - 1.0), r = 1.0 / am1;
        for (;;) {
            const double y = std::tan(pi * uniform01(eng));
            const double sy = s * y, t = sy + alpha;
            if (t <= 1.0) continue;  // x = s y + alpha - 1 <= 0
            const double x = t - 1.0;
            if (uniform01(eng) > (y * y + 1.0) * std::exp(std::log(x * r) * am1 - sy)) continue;
            return x;
        }
    }
    for (;;) {
        const double u = uniform01(eng);
        const double y = exponential(eng);
        double x, q;
        if (u < p) {
            x = std::exp(-(y * (1.0 / alpha)));
            q = p * std::exp(-x);
        } else {
            x = 1.0 + y;
            q = (1.0 - p) * std::pow(x, alpha - 1.0) + p;
        }
        if (u >= q) continue;
        return x;
    }
}

}  // namespace

// cvs: n_cv count vectors of M + 1 entries (-1 = omitted).  emit(sample, tpm[1..M], l_bar) for the nSpC samples of each
// vector in order; `sample` counts from 0 within this file.  Progress lines as calcCI.cpp:154 when `verbose`.
void ci_sample_vectors(const int32_t* cvs, int n_cv, int M, int nSpC, double pseudoC, uint32_t seed, const double* eel,
                       const double* mw, int thread_no, bool verbose,
                       const std::function<void(int64_t, const float*, float)>& emit) {
    std::mt19937 eng(seed);
    std::vector<double> theta(M + 1), alpha(M + 1), p(M + 1);
    std::vector<float> tpm(M + 1, 0.0f);  // entries with eel < EPSILON are never written and stay 0
    std::vector<char> draw(M + 1);
    const double e = std::exp(1.0);
    int64_t sample = 0;
    for (int c = 0; c < n_cv; ++c) {
        const int32_t* cvec = cvs + (size_t)c * (M + 1);
        for (int j = 0; j <= M; ++j) {
            draw[j] = j == 0 || (cvec[j] >= 0 && eel[j] >= kEps && mw[j] >= kEps);
            if (cvec[j] >= 0) {
                alpha[j] = cvec[j] + pseudoC;
                p[j] = e / (alpha[j] + e);
            }
        }
        for (int i = 0; i < nSpC; ++i) {
            double sum = 0.0;
            for (int j = 0; j <= M; ++j) {
                theta[j] = draw[j] ? gamma_draw(eng, alpha[j], p[j]) / mw[j] : 0.0;
                sum += theta[j];
            }
            if (!(sum >= kEps)) die("rsem-calculate-credibility-intervals: a sampled theta vector sums to 0");
            const double rs = 1.0 / sum;
            for (int j = 0; j <= M; ++j) theta[j] *= rs;

            sum = 0.0;
            for (int j = 1; j <= M; ++j)
                if (eel[j] >= kEps) {
                    tpm[j] = (float)(theta[j] / eel[j]);
                    sum += tpm[j];
                }
            if (!(sum >= kEps)) die("rsem-calculate-credibility-intervals: a sampled TPM vector sums to 0");
            const double rt = 1.0 / sum;
            float l_bar = 0.0f;
            for (int j = 1; j <= M; ++j) {
                const float t = (float)(tpm[j] * rt);
                l_bar = (float)(l_bar + t * eel[j]);
                tpm[j] = t * 1e6f;
            }
            emit(sample++, tpm.data() + 1, l_bar);
        }
        if (verbose && (c + 1) % 100 == 0) printf("Thread %d, %d count vectors are processed!\n", thread_no, c + 1);
    }
}

}  // namespace host
